"""Sharded sparse and TF-IDF search behind the C ABI (csrc/shard_group.cu): a group of shards must return what ONE index
holding every shard's rows at their global ids returns -- ids, counts and score bits -- with the same appends, deletes and
versions routed to the owning shard.  Sparse: thresholds, with and without the two-phase re-rank, deletes in several shards,
shards shorter than k, an empty shard, the device form.  TF-IDF: versioned op scripts, top_k None / 10 / 600, a term on one
shard only, bucket ties across shards with the later rank holding the smaller id.  One GPU: the shards share device 0 and
the gathers are the copy-based loopback; with >= 2 GPUs the same checks run over a real NCCL communicator."""
import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200.sharding import ShardGroup, shard_range
from tests import pysparse as ps
from tests import pytfidf as pt
from tests.sparse_data import slice_csr, zipf_csr
from tests.tfidf_data import op_script, query_csr, random_queries

pytestmark = pytest.mark.gpu


def devices(n):
    return list(range(n)) if cdb.device_count() >= n else [0] * n


def check(got, want):
    ids, scores, counts = got
    w_ids, w_scores, w_counts = want[:3]
    assert np.array_equal(counts, w_counts)
    assert np.array_equal(ids, w_ids)
    assert np.array_equal(np.ascontiguousarray(scores).view(np.uint32), np.ascontiguousarray(w_scores).view(np.uint32))


# ----------------------------------------------------------------------------- sparse
def sparse_group(corpus, bounds, bits=4, ub=1.0, slots=None):
    """shards over rows [bounds[r], bounds[r+1]) of corpus; slots[r] = the local slot of shard r"""
    n = len(bounds) - 1
    devs = devices(n)
    slots = list(range(n)) if slots is None else slots
    g = ShardGroup.local([devs[s] for s in range(n)])
    parts = []
    for r in range(n):
        b0, b1 = bounds[r], bounds[r + 1]
        base = b0 if b1 > b0 else bounds[-1] + r          # an empty shard: one row of capacity past every other range
        ix = cdb.SparseIndex(quantization_bits=bits, values_upper_bound=ub, capacity_rows=max(b1 - b0, 1),
                             capacity_pairs=int(corpus[0][b1] - corpus[0][b0]) + 8, id_base=base, device=devs[slots[r]])
        if b1 > b0:
            ix.append(slice_csr(corpus, b0, b1))
        g.attach_sparse(slots[r], ix)
        parts.append(ix)
    return g, parts


def whole_sparse(corpus, bits=4, ub=1.0):
    n = len(corpus[0]) - 1
    ix = cdb.SparseIndex(quantization_bits=bits, values_upper_bound=ub, capacity_rows=n, capacity_pairs=len(corpus[1]) + 8)
    ix.append(corpus)
    return ix


CASES = [(0.0, False, 10, 1), (0.5, False, 10, 1), (0.0, True, 10, 5), (0.5, True, 10, 5), (0.0, True, 1000, 5), (0.0, False, 1024, 1)]


@pytest.mark.parametrize("nshards", [2, 3])
def test_sparse_group_equals_the_whole_index(nshards):
    n, nq = 70000, 48
    corpus = zipf_csr(900 + nshards, n, vocab=3000, mean_pairs=24)
    queries = zipf_csr(950, nq, vocab=3000, mean_pairs=8)
    bounds = [shard_range(n, nshards, r)[0] for r in range(nshards)] + [n]
    g, parts = sparse_group(corpus, bounds)
    whole = whole_sparse(corpus)
    rng = np.random.default_rng(nshards)
    for step in range(2):
        for thr, rerank, k, f in CASES:
            opts = cdb.SparseSearchOptions(k, thr, rerank, f)
            check(g.search_sparse(queries, opts), whole.batch_search(queries, opts))
        # deletes in every shard, the first-ranked rows of some queries among them
        top = whole.batch_search(queries, cdb.SparseSearchOptions(3))[0][:4, 0]
        dead = np.unique(np.concatenate([rng.choice(n, 300, replace=False), top[top != cdb.INVALID_ID]])).astype(np.uint32)
        whole.delete_embedding(dead)
        for r, ix in enumerate(parts):
            mine = dead[(dead >= bounds[r]) & (dead < bounds[r + 1])] - bounds[r]
            assert mine.size
            ix.delete_embedding(mine)
    # a sample against the C oracle (whole corpus, deletes applied)
    deleted = whole.deleted_rows()[0]
    for thr, rerank, k, f in CASES[:4]:
        got = g.search_sparse(queries, cdb.SparseSearchOptions(k, thr, rerank, f))
        check(got, ps.search(corpus, queries, k, thr=thr, rerank=rerank, factor=f, deleted=deleted))
    g.close(); whole.close()
    for p in parts:
        p.close()


def test_sparse_short_and_empty_shards_and_rank_order():
    """shards of 5 / 0 / 8 rows (< k), attached in reverse slot order, quirky values at bits 6"""
    rows = [[(d % 5, float(v)) for d, v in zip(range(r % 4 + 1), np.linspace(0.1, 2.0, r % 4 + 1))] for r in range(13)]
    rows[2] = [(1, 0.0)]
    rows[3] = []
    corpus = cdb.sparse_csr(rows)
    bounds = [0, 5, 5, 13]
    g, parts = sparse_group(corpus, bounds, bits=6, ub=1.5, slots=[2, 1, 0])
    whole = whole_sparse(corpus, bits=6, ub=1.5)
    queries = [[(0, 1.0), (1, 0.5)], [(4, 2.0)], [(2, 0.3), (3, 0.3), (1, 0.01)], [], [(9, 1.0)]]
    for thr, rerank, k, f in [(0.0, False, 10, 1), (0.0, True, 10, 5), (0.0, True, 2, 2), (1.0, False, 3, 1), (0.0, True, 1, 1)]:
        opts = cdb.SparseSearchOptions(k, thr, rerank, f)
        got = g.search_sparse(queries, opts)
        check(got, whole.batch_search(queries, opts))
        check(got, ps.search(corpus, cdb.sparse_csr(queries), k, bits=6, ub=1.5, thr=thr, rerank=rerank, factor=f))
    g.close(); whole.close()
    for p in parts:
        p.close()


def test_sparse_rerank_is_two_phase():
    """k = 1, f = 2: shard 0's rows 0 and 1 hold the group's top 2 by similarity (ties to the smaller id); shard 1's rows
    have the same similarity but a larger raw value.  Re-ranking each shard's own top 2 would return id 10."""
    rows = [[(0, 1.0)], [(0, 1.0)]] + [[]] * 8 + [[(0, 5.0)], [(0, 5.0)]]
    corpus = cdb.sparse_csr(rows)
    g, parts = sparse_group(corpus, [0, 10, 12])
    opts = cdb.SparseSearchOptions(1, 0.0, True, 2)
    ids, scores, counts = g.search_sparse([[(0, 1.0)]], opts)
    assert ids[0, 0] == 0 and scores[0, 0] == 1.0 and counts[0] == 1
    check((ids, scores, counts), ps.search(corpus, cdb.sparse_csr([[(0, 1.0)]]), 1, rerank=True, factor=2))
    g.close()
    for p in parts:
        p.close()


def test_sparse_rank_group_of_one_and_device_form():
    import torch
    n, nq = 40000, 33
    corpus = zipf_csr(970, n, vocab=2000, mean_pairs=16)
    queries = zipf_csr(971, nq, vocab=2000, mean_pairs=6)
    g = ShardGroup.rank(None, 1, 0, 0)
    ix = cdb.SparseIndex(capacity_rows=n, capacity_pairs=len(corpus[1]) + 8)
    ix.append(corpus)
    g.attach_sparse(0, ix)
    dev = torch.device("cuda", 0)
    o, d, v = [torch.from_numpy(a.astype(t)).to(dev) for a, t in zip(queries, (np.int64, np.int32, np.float32))]
    s = torch.cuda.Stream(dev)
    for thr, rerank, k, f in CASES:
        opts = cdb.SparseSearchOptions(k, thr, rerank, f)
        host = g.search_sparse(queries, opts)
        check(host, ix.batch_search(queries, opts))
        ids = torch.zeros((nq, k), dtype=torch.int32, device=dev)
        sc = torch.zeros((nq, k), dtype=torch.float32, device=dev)
        cnt = torch.zeros(nq, dtype=torch.int32, device=dev)
        with torch.cuda.stream(s):
            g.search_sparse_device(o.data_ptr(), d.data_ptr(), v.data_ptr(), nq, opts, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                                   s.cuda_stream)
        s.synchronize()
        check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), host)
    g.close(); ix.close()


def test_sparse_attach_and_search_refusals():
    devs = devices(2)
    g = ShardGroup.local(devs)
    a = cdb.SparseIndex(capacity_rows=100, capacity_pairs=100, id_base=0, device=devs[0])
    opts = cdb.SparseSearchOptions(5)
    with pytest.raises(cdb.CosdataError):           # slot 1 has no sparse shard
        g.search_sparse([[(0, 1.0)]], opts)
    g.attach_sparse(0, a)
    for kw in (dict(quantization_bits=5), dict(values_upper_bound=2.0), dict(id_base=50)):
        b = cdb.SparseIndex(**{**dict(capacity_rows=100, capacity_pairs=100, id_base=100, device=devs[1]), **kw})
        with pytest.raises(cdb.CosdataError):
            g.attach_sparse(1, b)
        b.close()
    if cdb.device_count() >= 2:
        b = cdb.SparseIndex(capacity_rows=100, capacity_pairs=100, id_base=100, device=0)
        with pytest.raises(cdb.CosdataError):
            g.attach_sparse(1, b)
        b.close()
    b = cdb.SparseIndex(capacity_rows=100, capacity_pairs=100, id_base=100, device=devs[1])
    g.attach_sparse(1, b)
    for bad in (cdb.SparseSearchOptions(0), cdb.SparseSearchOptions(1025), cdb.SparseSearchOptions(1024, rerank=True, reranking_factor=6)):
        with pytest.raises(cdb.CosdataError):
            g.search_sparse([[(0, 1.0)]], bad)
    ids, _, counts = g.search_sparse([[(0, 1.0)]], opts)
    assert counts[0] == 0 and (ids == cdb.INVALID_ID).all()
    t = cdb.TfIdfIndex(capacity_rows=10, capacity_pairs=10, device=devs[0])
    g.attach_tfidf(0, t)
    with pytest.raises(cdb.CosdataError):           # slot 1 has no tf-idf shard
        g.search_tfidf([[1]])
    t2 = cdb.TfIdfIndex(capacity_rows=10, capacity_pairs=10, id_base=5, device=devs[1])
    with pytest.raises(cdb.CosdataError):           # ids 5..14 meet 0..9
        g.attach_tfidf(1, t2)
    g.close()
    for x in (a, b, t, t2):
        x.close()


# ----------------------------------------------------------------------------- TF-IDF
class Routed:
    """a TF-IDF shard group over fixed global id ranges [bounds[r], bounds[r+1]) next to one whole index and the C
    oracle; appends and deletes go to the whole index and to the owning shards with the same versions"""

    def __init__(self, bounds, slots=None):
        n = len(bounds) - 1
        devs = devices(n)
        slots = list(range(n)) if slots is None else slots
        self.bounds = bounds
        self.g = ShardGroup.local(devs)
        self.parts = []
        for r in range(n):
            ix = cdb.TfIdfIndex(capacity_rows=bounds[r + 1] - bounds[r], capacity_pairs=1 << 14, id_base=bounds[r], device=devs[slots[r]])
            self.g.attach_tfidf(slots[r], ix)
            self.parts.append(ix)
        self.whole = cdb.TfIdfIndex(capacity_rows=bounds[-1], capacity_pairs=1 << 16)
        self.orc = pt.Oracle()
        self.n = 0

    def append(self, rows, counted, version):
        counted = np.ones(len(rows), np.uint8) if counted is None else np.asarray(counted, np.uint8)
        self.whole.append(rows, version, counted)
        self.orc.append(cdb.sparse_csr(rows), version, counted)
        for r, ix in enumerate(self.parts):
            a, b = max(self.n, self.bounds[r]), min(self.n + len(rows), self.bounds[r + 1])
            if a < b:
                ix.append(rows[a - self.n:b - self.n], version, counted[a - self.n:b - self.n])
        self.n += len(rows)

    def delete(self, rows, version):
        rows = np.asarray(rows, np.uint32)
        self.whole.delete_embedding(rows, version)
        self.orc.delete(rows, version)
        for r, ix in enumerate(self.parts):
            mine = rows[(rows >= self.bounds[r]) & (rows < self.bounds[r + 1])]
            if mine.size:
                ix.delete_embedding(mine - self.bounds[r], version)

    def check(self, qs, ks=(0, 10, 600), oracle=False):
        for k in ks:
            got = self.g.search_tfidf(qs, k)
            check(got, self.whole.batch_search(qs, k))
            if oracle:
                check(got, self.orc.search(query_csr(qs), k))

    def close(self):
        self.g.close()
        for x in self.parts + [self.whole]:
            x.close()
        self.orc.close()


@pytest.mark.parametrize("seed", range(4))
def test_tfidf_group_follows_versioned_op_scripts(seed):
    vocab, ops = op_script(seed, steps=10, vocab_size=12, rows_per_step=40)
    nshards = 2 + seed % 2
    grp = Routed([0, 70, 140, 1000][:nshards] + [1000], slots=list(range(nshards))[::-1] if seed % 2 else None)
    qs = random_queries(np.random.default_rng(seed), vocab, 40) + [[]]
    for i, op in enumerate(ops):
        if op[0] == "append":
            grp.append(op[1], op[2], op[3])
        else:
            grp.delete(op[1], op[2])
        grp.check(qs, oracle=i % 3 == 0)
    grp.close()


def test_tfidf_term_on_one_shard_and_cross_shard_bucket_ties():
    """slot 0 holds ids 1000.., slot 1 ids 0..: the later rank holds the smaller id.  Ids 5 and 1029 share bucket 5 with
    equal scores, ids 7 and 1031 with +0 and -0; term 77 lives on slot 0's shard only."""
    grp = Routed([0, 1000, 1200], slots=[1, 0])
    rows = [[] for _ in range(1100)]
    counted = np.zeros(1100, np.uint8)
    for r, row in ((5, [(1, 2.0)]), (1029, [(1, 2.0)]), (7, [(2, -0.0)]), (1031, [(2, 0.0)]), (9, [(1, 1.0), (2, 3.0)]),
                   (1040, [(77, 1.5), (1, 0.5)]), (1041, [(1, 2.0)]), (12, [(3, 1.0)])):
        rows[r] = row
        counted[r] = 1
    grp.append(rows[:600], counted[:600], 1)
    grp.append(rows[600:], counted[600:], 2)
    qs = [[1], [2], [77], [77, 1], [1, 2, 3], [3, 77], [99]]
    grp.check(qs, ks=(0, 1, 2, 10, 600), oracle=True)
    ids, scores, counts = grp.g.search_tfidf([[1]], 10)
    assert 5 in ids[0] and 1029 not in ids[0]
    ids, scores, counts = grp.g.search_tfidf([[2]], 10)
    assert 7 in ids[0] and 1031 not in ids[0]
    grp.delete([5], 2)
    grp.check(qs, oracle=True)
    grp.close()
