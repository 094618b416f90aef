"""Sparse and TF-IDF search at the limits of their host plans, against the CPU oracles (tests/sparse_oracle.c,
tests/tfidf_oracle.c) and, for shard groups, against one index holding every row: ids, counts and score bits exact.

The plans (tests/text_plan.py): sparse merge trees of two and three levels with groups of one list, query chunks after the
first (q0 > 0) up to the 65,535-query grid limit, queries longer than one 512-pair scoring pass, and shard groups wider than
one merge group, both across the ranks and inside a shard.  Every case asserts that a single-threaded search launched
exactly the kernels of the plan it names, so none can quietly take a shallower path.

The deep-tree corpus has short rows (1-4 pairs) over four hot dims and a few value levels: every tile has far more touched
rows than any m, and the cut at m falls inside long runs of equal similarities spread over every tile, so every merge
decides on id bits across lists.  One tile is wholly deleted (a list of count 0), the last holds fewer than m rows, and the
largest index sits at the top of the id space (its last id is 0xFFFFFFFE)."""
import functools

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200.sharding import ShardGroup
from tests import pysparse as ps
from tests import pytfidf as pt
from tests import text_plan as tp
from tests.sparse_data import concat_csr, quirky_rows, slice_csr
from tests.test_gpu_sharded_text import Routed, devices
from tests.tfidf_data import query_csr, random_queries, random_rows

pytestmark = pytest.mark.gpu

T = tp.TILE_ROWS
N26 = 25 * T + 700                 # 26 tiles, the last with 700 rows: fewer than any m of these cases
HI_BASE = (1 << 32) - 1 - N26      # capacity_rows = N26, so the last id is 0xFFFFFFFE
DEAD_TILE = 7
HOT = 4
LEVELS = np.array([0.05, 0.2, 0.4, 0.6, 0.8, 1.0], np.float32)     # keys 0, 3, 6, 9, 12, 15 at bits 4, ub 1.0
LEVEL_P = [0.5, 0.25, 0.15, 0.07, 0.025, 0.005]                     # the high similarities are rare, the ties long
LAST_DIM = 5000                    # held by the last row only


def check(got, want):
    ids, scores, counts = got
    w_ids, w_scores, w_counts = want[:3]
    assert np.array_equal(counts, w_counts)
    assert np.array_equal(ids, w_ids)
    assert np.array_equal(np.ascontiguousarray(scores).view(np.uint32), np.ascontiguousarray(w_scores).view(np.uint32))


def check_rows(got, want, rows):
    check(tuple(a[rows] for a in got[:3]), want)


def launches(fn):
    """(fn(), the kernel launches it made); the callers search from one thread"""
    before = cdb.kernel_launch_count()
    out = fn()
    return out, cdb.kernel_launch_count() - before


def chunk_edges(sizes, every=0):
    """the first and last query of every chunk, plus every `every`-th query"""
    out, q0 = set(), 0
    for c in sizes:
        out |= {q0, q0 + c - 1}
        q0 += c
    if every:
        out |= set(range(0, q0, every))
    return np.array(sorted(out))


def pick(csr, rows):
    return concat_csr([slice_csr(csr, int(i), int(i) + 1) for i in rows])


# ----------------------------------------------------------------------------- corpora
@functools.lru_cache(maxsize=None)
def short_corpus():
    """N26 rows of 1-4 pairs: the first a hot dim (0..3) in 95% of rows, the rest cold dims; values on LEVELS"""
    rng = np.random.default_rng(2024)
    lens = rng.integers(1, 5, N26)
    off = np.zeros(N26 + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    total = int(off[-1])
    dims = rng.integers(HOT, 3000, total).astype(np.uint32)
    hot = rng.random(N26) < 0.95
    dims[off[:-1].astype(np.int64)[hot]] = rng.integers(0, HOT, int(hot.sum())).astype(np.uint32)
    vals = LEVELS[rng.choice(len(LEVELS), total, p=LEVEL_P)]
    dims[-1] = LAST_DIM
    return off, dims, vals


@functools.lru_cache(maxsize=None)
def short_queries(nq=1500):
    """2-4 distinct hot dims and 0-2 cold dims per query"""
    rng = np.random.default_rng(77)
    rows = []
    for _ in range(nq):
        h = rng.choice(HOT, int(rng.integers(2, HOT + 1)), replace=False)
        q = [(int(d), float(rng.choice([0.3, 0.6, 0.8, 1.0]))) for d in h]
        q += [(int(rng.integers(HOT, 3000)), float(rng.random())) for _ in range(int(rng.integers(0, 3)))]
        rows.append(q)
    return cdb.sparse_csr(rows)


def similarities(corpus, query, deleted):
    """the u32 similarity of every live touched row to one query (bits 4, ub 1.0, no threshold), -1 elsewhere; the
    similarities of the short corpus stay far below 2^24"""
    off, dims, vals = corpus
    row = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    levels, inv = np.unique(vals, return_inverse=True)
    keys = np.array([ps.quantize(v, 1.0, 4) for v in levels], np.int64)[inv]
    sim = np.zeros(len(off) - 1, np.int64)
    touched = np.zeros(len(off) - 1, bool)
    for d, v in zip(query[1].tolist(), query[2].tolist()):
        hit = dims == d
        np.add.at(sim, row[hit], keys[hit] * ps.quantize(v, 1.0, 4))
        touched[row[hit]] = True
    return np.where(touched & (deleted == 0), sim, -1).astype(np.float32)


def dead_rows(n):
    """a whole tile and every 101st row"""
    d = np.zeros(n, np.uint8)
    if n > (DEAD_TILE + 1) * T:
        d[DEAD_TILE * T:(DEAD_TILE + 1) * T] = 1
    d[5::101] = 1
    return d


# (rows, id_base, deletes) of the indexes over prefixes of the short corpus
SHORT_INDEXES = {"t26": (N26, HI_BASE, True), "t5": (5 * T - 123, 0, False), "t6": (5 * T + 4000, 11, True),
                 "t7": (7 * T - 1, 3, False)}


@pytest.fixture(scope="module")
def short_ix():
    made = {}

    def get(name):
        if name not in made:
            n, base, dels = SHORT_INDEXES[name]
            corpus = slice_csr(short_corpus(), 0, n)
            ix = cdb.SparseIndex(quantization_bits=4, values_upper_bound=1.0, capacity_rows=n, capacity_pairs=len(corpus[1]),
                                 id_base=base)
            ix.append(corpus)
            deleted = dead_rows(n) if dels else np.zeros(n, np.uint8)
            if dels:
                ix.delete_embedding(np.flatnonzero(deleted).astype(np.uint32))
            made[name] = (ix, corpus, base, deleted)
        return made[name]

    yield get
    for ix, *_ in made.values():
        ix.close()


# ----------------------------------------------------------------------------- 1, 2: merge trees and query chunks
TREE_CASES = [
    # index, k, rerank, factor, nq, merge levels, chunks
    ("t26", 1024, False, 1, 500, [2, 1], [500]),          # g = 25: a last group of one list
    ("t26", 1024, True, 5, 500, [6, 2, 1], [409, 91]),    # g = 5
    ("t26", 1000, True, 5, 500, [6, 2, 1], [419, 81]),
    ("t5", 1024, True, 5, 64, [1], [64]),                 # one full group
    ("t6", 1024, True, 5, 64, [2, 1], [64]),              # a group of one
    ("t6", 1024, False, 1, 64, [1], [64]),
    ("t7", 1024, True, 5, 1500, [2, 1], [1456, 44]),
    ("t7", 600, False, 1, 1500, [1], [1500]),
]


@pytest.mark.parametrize("name,k,rerank,factor,nq,levels,sizes", TREE_CASES)
def test_merge_trees_and_chunks_against_the_oracle(short_ix, name, k, rerank, factor, nq, levels, sizes):
    ix, corpus, base, deleted = short_ix(name)
    n_tiles = tp.n_tiles(len(corpus[0]) - 1)
    m = k * factor
    assert tp.tree_levels(n_tiles, m) == levels and tp.chunks(nq, tp.sparse_chunk(nq, n_tiles, m)) == sizes
    queries = slice_csr(short_queries(), 0, nq)
    opts = cdb.SparseSearchOptions(k, 0.0, rerank, factor)
    got, n = launches(lambda: ix.batch_search(queries, opts))
    sample = chunk_edges(sizes, every=97) if n_tiles > 7 else np.arange(nq) if nq <= 64 else chunk_edges(sizes, every=37)
    want = ps.search(corpus, pick(queries, sample), k, bits=4, ub=1.0, rerank=rerank, factor=factor, id_base=base, deleted=deleted)
    check_rows(got, want, sample)
    assert n == tp.sparse_launches(nq, n_tiles, m) == len(sizes) * (2 + len(levels))
    # the cut at m lies inside a run of equal similarities held by rows of several tiles
    if not rerank and name == "t26":
        q = int(sample[0])
        sims = similarities(corpus, slice_csr(queries, q, q + 1), deleted)
        run = np.flatnonzero(sims == np.float32(got[1][q, k - 1]))
        assert np.unique(run // T).size > 1 and run.size > np.count_nonzero(got[1][q] == got[1][q, k - 1])
    if name == "t26":
        assert (got[0] != cdb.INVALID_ID).all()           # every query fills k from the 2^32 - 2 - N26 .. 2^32 - 2 range
        dead_ids = np.uint32(base) + np.arange(DEAD_TILE * T, (DEAD_TILE + 1) * T, dtype=np.uint32)
        assert not np.isin(got[0], dead_ids).any()


def test_last_id_of_the_id_space_is_found(short_ix):
    """a dim only the last row holds: id 0xFFFFFFFE, whose inverted id in the selection key is 1"""
    ix, corpus, base, deleted = short_ix("t26")
    assert base + N26 - 1 == 0xFFFFFFFE
    queries = cdb.sparse_csr([[(LAST_DIM, 1.0)], [(LAST_DIM, 0.0), (0, 1.0)], [(LAST_DIM + 1, 1.0)]])
    for k, rerank in ((3, False), (1024, True)):
        got, n = launches(lambda: ix.batch_search(queries, cdb.SparseSearchOptions(k, 0.0, rerank, 5)))
        assert n == tp.sparse_launches(3, 26, k * (5 if rerank else 1))
        assert got[0][0, 0] == 0xFFFFFFFE and got[2][0] == 1 and got[2][2] == 0
        check(got, ps.search(corpus, queries, k, id_base=base, rerank=rerank, factor=5, deleted=deleted))


def test_device_entry_point_chunks_on_a_side_stream(short_ix):
    """t7, nq = 1500 at m = 5120 (chunks of 1456 + 44) through cdb_sparse_search_batch_device on a side stream"""
    import ctypes as C

    import torch
    from cosdata_b200 import _lib
    ix, *_ = short_ix("t7")
    queries = short_queries()
    nq, k = 1500, 1024
    opts = cdb.SparseSearchOptions(k, 0.0, True, 5)
    host = ix.batch_search(queries, opts)
    dev = torch.device("cuda", 0)
    o, d, v = [torch.from_numpy(a.astype(t)).to(dev) for a, t in zip(queries, (np.int64, np.int32, np.float32))]
    ids = torch.full((nq, k), 7, dtype=torch.int32, device=dev)
    sc = torch.full((nq, k), 7.0, dtype=torch.float32, device=dev)
    cnt = torch.full((nq,), 7, dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)
    s = torch.cuda.Stream(dev)
    p = opts.params()
    rc, n = launches(lambda: _lib.load().cdb_sparse_search_batch_device(ix.h, o.data_ptr(), d.data_ptr(), v.data_ptr(), nq, C.byref(p),
                                                                        ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                                                                        C.c_void_p(s.cuda_stream)))
    assert rc == 0 and n == tp.sparse_launches(nq, 7, 5120) == 2 * 4
    s.synchronize()
    check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), host)


# ----------------------------------------------------------------------------- 2: the grid limit
GRID_NQ = 70_000


@functools.lru_cache(maxsize=None)
def grid_sparse():
    corpus = cdb.sparse_csr(quirky_rows(5, 2000, 60))
    queries = cdb.sparse_csr(quirky_rows(6, GRID_NQ, 64, max_len=4))     # dims 60..63 are absent
    return corpus, queries


@pytest.mark.parametrize("k,rerank", [(10, False), (10, True)])
def test_sparse_grid_limit_chunks(k, rerank):
    corpus, queries = grid_sparse()
    ix = cdb.SparseIndex(quantization_bits=5, values_upper_bound=1.5, capacity_rows=2000, capacity_pairs=len(corpus[1]), id_base=9)
    ix.append(corpus)
    m = k * (5 if rerank else 1)
    assert tp.chunks(GRID_NQ, tp.sparse_chunk(GRID_NQ, 1, m)) == [65535, 4465]
    got, n = launches(lambda: ix.batch_search(queries, cdb.SparseSearchOptions(k, 0.0, rerank, 5)))
    assert n == tp.sparse_launches(GRID_NQ, 1, m) == 2 * 2
    check(got, ps.search(corpus, queries, k, bits=5, ub=1.5, rerank=rerank, factor=5, id_base=9))
    ix.close()


@pytest.mark.parametrize("k", [10, 0])
def test_tfidf_grid_limit_chunks(k):
    rng = np.random.default_rng(8)
    vocab = rng.choice(1 << 31, 300, replace=False).astype(np.uint32)
    rows, counted = random_rows(rng, 2000, vocab, max_terms=8)
    ix = cdb.TfIdfIndex(capacity_rows=2000, capacity_pairs=1 << 16, id_base=77)
    orc = pt.Oracle(77)
    ix.append(rows, 1, counted)
    orc.append(cdb.sparse_csr(rows), 1, counted)
    queries = query_csr(random_queries(np.random.default_rng(9), vocab, GRID_NQ, max_terms=4))
    assert tp.chunks(GRID_NQ, tp.tfidf_chunk(GRID_NQ, 1)) == [65535, 4465]
    got, n = launches(lambda: ix.batch_search(queries, k))
    assert n == tp.tfidf_launches(GRID_NQ, 1) == 2 * 2
    check(got, orc.search(queries, k))
    ix.close()
    orc.close()


# ----------------------------------------------------------------------------- 3: long queries
LONG_N = 40_000
LONG_LENS = (511, 512, 513, 1025, 3000)


@functools.lru_cache(maxsize=None)
def long_corpus():
    """2 tiles of 1-12 pairs over dims 1..3999 at bits 8; 100 rows hold dim 0 at 1.0 sixty to eighty times, so the
    3000-pair query's 1500 pairs of dim 0 give similarities past 2^32"""
    rng = np.random.default_rng(31)
    rows = []
    for r in range(LONG_N):
        m = int(rng.integers(1, 13))
        row = list(zip(rng.integers(1, 4000, m).tolist(), (rng.random(m) * 1.2).astype(np.float32).tolist()))
        if r % 400 == 7:
            row = [(0, 1.0)] * int(rng.integers(60, 81)) + row
        rows.append(row)
    rows[11] = [(3, 0.0), (3, float("nan")), (5, -1.0)]
    return cdb.sparse_csr(rows)


@functools.lru_cache(maxsize=None)
def long_queries():
    rng = np.random.default_rng(32)
    out = []
    for n in LONG_LENS:
        dims = rng.integers(1, 4000, n).astype(np.uint32)
        vals = (rng.random(n) * 1.2).astype(np.float32)
        dims[rng.random(n) < 0.05] = rng.integers(5000, 6000)       # a dim absent from the index
        vals[rng.random(n) < 0.2] = np.float32(0.1)             # qv 25 <= low: only keys >= etv under a threshold of 0.3
        sp = rng.random(n) < 0.06
        vals[sp] = np.array([0.0, -0.7, np.nan], np.float32)[rng.integers(0, 3, int(sp.sum()))]
        if n == 3000:
            hot = rng.random(n) < 0.5
            dims[hot], vals[hot] = 0, np.float32(1.0)
        for b in range(512, n + 2, 512):                         # one dim on both sides of every pass boundary
            dims[b - 2:b + 2] = dims[b - 2]
        out.append(list(zip(dims.tolist(), vals.tolist())))
    return cdb.sparse_csr(out)


@pytest.fixture(scope="module")
def long_ix():
    corpus = long_corpus()
    ix = cdb.SparseIndex(quantization_bits=8, values_upper_bound=1.0, capacity_rows=LONG_N, capacity_pairs=len(corpus[1]))
    ix.append(corpus)
    yield ix, corpus
    ix.close()


def test_long_query_similarities_wrap():
    """every row holding dim 0 has a similarity past 2^32 to the 3000-pair query: 255 * 255 per pair of dim 0 on each side"""
    corpus, q = long_corpus(), long_queries()
    n_hot = int((q[1][int(q[0][4]):int(q[0][5])] == 0).sum())
    copies = [int((corpus[1][int(corpus[0][r]):int(corpus[0][r + 1])] == 0).sum()) for r in range(7, LONG_N, 400)]
    assert n_hot * 255 * 255 * min(copies) > 1 << 32


@pytest.mark.parametrize("thr", [0.0, 0.3])
@pytest.mark.parametrize("k,rerank", [(100, False), (100, True), (1024, False)])
def test_long_sparse_queries_top_k(long_ix, thr, k, rerank):
    ix, corpus = long_ix
    queries = long_queries()
    m = k * (5 if rerank else 1)
    got, n = launches(lambda: ix.batch_search(queries, cdb.SparseSearchOptions(k, thr, rerank, 5)))
    assert n == tp.sparse_launches(len(LONG_LENS), 2, m)
    check(got, ps.search(corpus, queries, k, bits=8, ub=1.0, thr=thr, rerank=rerank, factor=5))


@pytest.mark.parametrize("thr,rerank", [(0.0, False), (0.3, True)])
def test_long_sparse_queries_top_k_none(long_ix, thr, rerank):
    ix, corpus = long_ix
    queries = long_queries()
    off, ids, scores = ix.batch_search_all(queries, cdb.SparseSearchOptions(None, thr, rerank))
    w_ids, w_scores, w_counts = ps.search(corpus, queries, LONG_N, bits=8, ub=1.0, thr=thr, rerank=rerank, factor=1)
    assert np.array_equal(np.diff(off.astype(np.int64)), w_counts.astype(np.int64))
    for q in range(len(LONG_LENS)):
        b, e, c = int(off[q]), int(off[q + 1]), int(w_counts[q])
        assert np.array_equal(ids[b:e], w_ids[q, :c]), q
        assert np.array_equal(scores[b:e].view(np.uint32), w_scores[q, :c].view(np.uint32)), q


def sparse_group(corpus, bounds, base, bits, ub, deleted=None):
    """one-device (loopback) group over rows [bounds[r], bounds[r+1]) at ids base + bounds[r]; an empty range gets one id
    of capacity just below base"""
    g = ShardGroup.local([0] * (len(bounds) - 1))
    parts = []
    for r in range(len(bounds) - 1):
        b0, b1 = bounds[r], bounds[r + 1]
        ix = cdb.SparseIndex(quantization_bits=bits, values_upper_bound=ub, capacity_rows=max(b1 - b0, 1),
                             capacity_pairs=int(corpus[0][b1] - corpus[0][b0]) + 8, id_base=base + b0 if b1 > b0 else base - 1)
        if b1 > b0:
            ix.append(slice_csr(corpus, b0, b1))
            if deleted is not None and deleted[b0:b1].any():
                ix.delete_embedding(np.flatnonzero(deleted[b0:b1]).astype(np.uint32))
        g.attach_sparse(r, ix)
        parts.append(ix)
    return g, parts


def close_group(g, parts):
    g.close()
    for p in parts:
        p.close()


@pytest.mark.parametrize("thr", [0.0, 0.3])
def test_long_sparse_queries_in_a_group_of_three(long_ix, thr):
    ix, corpus = long_ix
    queries = long_queries()
    bounds = [0, 13_000, 26_000, LONG_N]
    g, parts = sparse_group(corpus, bounds, 0, 8, 1.0)
    for k, rerank in ((100, False), (100, True)):
        opts = cdb.SparseSearchOptions(k, thr, rerank, 5)
        got, n = launches(lambda: g.search_sparse(queries, opts))
        assert n == tp.sparse_group_launches(len(LONG_LENS), [1, 1, 1], k * (5 if rerank else 1), rerank)
        check(got, ix.batch_search(queries, opts))
        check(got, ps.search(corpus, queries, k, bits=8, ub=1.0, thr=thr, rerank=rerank, factor=5))
    close_group(g, parts)


@functools.lru_cache(maxsize=None)
def long_tfidf():
    """3000 rows over a 2000-hash vocabulary and queries of 512, 513 and 1500 terms: repeated hashes on both sides of every
    512-term boundary, absent hashes"""
    rng = np.random.default_rng(41)
    vocab = rng.choice(1 << 31, 2000, replace=False).astype(np.uint32)
    rows, counted = random_rows(rng, 3000, vocab, max_terms=12, uncounted=0.05)
    qs = []
    for n in (512, 513, 1500):
        q = rng.choice(vocab, n).astype(np.uint32)
        q[rng.random(n) < 0.05] = rng.integers(1 << 31, 1 << 32, dtype=np.uint64).astype(np.uint32)
        for b in range(512, n + 2, 512):
            q[b - 2:b + 2] = q[b - 2]
        qs.append(q.tolist())
    return rows, counted, qs


@pytest.mark.parametrize("k", [10, 0])
def test_long_tfidf_queries(k):
    rows, counted, qs = long_tfidf()
    ix = cdb.TfIdfIndex(capacity_rows=3000, capacity_pairs=1 << 16, id_base=5)
    orc = pt.Oracle(5)
    ix.append(rows, 2, counted)
    orc.append(cdb.sparse_csr(rows), 2, counted)
    got, n = launches(lambda: ix.batch_search(query_csr(qs), k))
    assert n == tp.tfidf_launches(len(qs), 1)
    check(got, orc.search(query_csr(qs), k))
    ix.close()
    orc.close()


def test_long_tfidf_queries_in_a_group_of_three_with_the_idf_step():
    """the shards score with the group's idf of every query term, q_idf[j0 + tid], in every 512-term pass; the host form
    launches the group's idf step (a statistics kernel per slot, the idf kernel) before the scoring"""
    rows, counted, qs = long_tfidf()
    grp = Routed([0, 1000, 2000, 3000])
    grp.append(rows, counted, 2)
    for k in (10, 0):
        got, n = launches(lambda: grp.g.search_tfidf(query_csr(qs), k))
        assert n == tp.tfidf_group_search_launches(len(qs), [1, 1, 1], sum(map(len, qs)), len(set(devices(3))) < 3)
        check(got, grp.whole.batch_search(query_csr(qs), k))
        check(got, grp.orc.search(query_csr(qs), k))
    grp.close()


# ----------------------------------------------------------------------------- 4: shard groups wider than one merge group
GROUP_NQ = 900
GROUP_CASES = [(1000, True, 5), (1024, True, 5), (1024, False, 1)]


def wide_bounds(world):
    """an 11-tile shard, an empty one, and the rest of the short corpus over world - 2 shards"""
    rest = np.linspace(11 * T, N26, world - 1).astype(int).tolist()
    return [0, 11 * T] + rest


@pytest.mark.parametrize("world", [6, 8])
def test_wide_sparse_groups(short_ix, world):
    whole, corpus, base, deleted = short_ix("t26")
    bounds = wide_bounds(world)
    assert len(bounds) == world + 1 and bounds[1] == bounds[2]
    tiles = [tp.n_tiles(b1 - b0) for b0, b1 in zip(bounds, bounds[1:])]
    g, parts = sparse_group(corpus, bounds, base, 4, 1.0, deleted)
    queries = slice_csr(short_queries(), 0, GROUP_NQ)
    for k, rerank, f in GROUP_CASES:
        m = k * f
        gsizes = tp.chunks(GROUP_NQ, tp.group_chunk(GROUP_NQ, world, m * 8 + 4))
        if rerank:
            assert tp.merge_lists_levels(world, m) == [2, 1] and tp.merge_lists_levels(11, m) == [3, 1]
            assert len(tp.chunks(gsizes[0], tp.shard_select_chunk(gsizes[0], 11, m))) == 2
        opts = cdb.SparseSearchOptions(k, 0.0, rerank, f)
        got, n = launches(lambda: g.search_sparse(queries, opts))
        assert n == tp.sparse_group_launches(GROUP_NQ, tiles, m, rerank)
        check(got, whole.batch_search(queries, opts))
        sample = chunk_edges(gsizes, every=211)
        sample = np.union1d(sample, chunk_edges(tp.chunks(gsizes[0], tp.shard_select_chunk(gsizes[0], 11, m))))
        want = ps.search(corpus, pick(queries, sample), k, bits=4, ub=1.0, rerank=rerank, factor=f, id_base=base, deleted=deleted)
        check_rows(got, want, sample)
    close_group(g, parts)


def test_tfidf_group_of_eight_bucket_ties_across_ranks_with_the_idf_step():
    """shard r (ids 600r..) sits in slot 7 - r, so later ranks hold smaller ids.  Every id = 5 (mod 512) holds the same row:
    one tie per bucket across ranks, won by id 5 on the last rank; ids = 7 (mod 512) tie at +0 and -0.  The launch count
    includes the group's idf step."""
    rng = np.random.default_rng(12)
    vocab = rng.choice(1 << 30, 40, replace=False).astype(np.uint32)
    h1, h2 = (1 << 30) + 1, (1 << 30) + 2
    rows, counted = random_rows(rng, 4800, vocab, max_terms=5)
    for r in range(4800):
        if r % 512 == 5:
            rows[r], counted[r] = [(h1, 2.0)], 1
        elif r % 512 == 7:
            rows[r], counted[r] = [(h2, 0.0 if (r // 512) % 2 else -0.0), (int(vocab[0]), 0.5)], 1
    grp = Routed(list(range(0, 4801, 600)), slots=list(range(8))[::-1])
    grp.append(rows[:2500], counted[:2500], 1)
    grp.append(rows[2500:], counted[2500:], 2)
    grp.delete(np.arange(3, 4800, 37, dtype=np.uint32), 2)
    qs = [[h1], [h2], [h1, h2], [h2, int(vocab[0])]] + random_queries(np.random.default_rng(13), np.concatenate([vocab, [h1, h2]]), 60)
    for k in (0, 1, 10, 600):
        got, n = launches(lambda: grp.g.search_tfidf(query_csr(qs), k))
        assert n == tp.tfidf_group_search_launches(len(qs), [1] * 8, sum(map(len, qs)), len(set(devices(8))) < 8)
        check(got, grp.whole.batch_search(query_csr(qs), k))
        check(got, grp.orc.search(query_csr(qs), k))
    ids = grp.g.search_tfidf([[h1]], 10)[0][0]
    assert 5 in ids and 517 not in ids and 1029 not in ids
    ids, scores, _ = grp.g.search_tfidf([[h2]], 0)
    assert 7 in ids[0] and 519 not in ids[0]
    grp.close()
