"""Hybrid search over mixed batches (cdb_hybrid_search_batch_mixed[_sharded][_device]) on the GPU, bit for bit on ids,
counts and score bits:
  * every row equals the two-source entry point's row for that query when the batch is split by kind (the split-by-kind
    calls, reassembled in request order), and tests/pyhybrid_mixed.fuse_mixed over each source's own search of its batch;
  * batches of one kind, two kinds, all three shuffled, B = 1, a source with no queries, and dense searches that set error
    flags (the bytes land at the positions of the queries that name dense; sparse + TF-IDF queries get 0);
  * single index (host and device forms), a 2-slot loopback group (host and device forms, the device form with a TF-IDF
    source against the host form), a one-slot group over a replica graph with dense_id_stride, and a group batch above
    one fusion chunk;
  * each source is searched once per call: the kernel launches are those of the three sub-searches plus one fusion per
    kind present."""
import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200.sharding import ShardGroup, shard_range
from tests import pyhybrid as ph
from tests import pyhybrid_mixed as pm
from tests.sparse_data import slice_csr, zipf_csr
from tests.tfidf_data import zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu
N, DIM, BMAX, VOCAB = 20_000, 64, 1024, 3000
DENSE_HNSW = {"mode": cdb.SearchMode.HNSW, "ef_search": 256, "shortlist_size": 64}
DENSE_TC = {"mode": cdb.SearchMode.BRUTE_RAW, "tensor_with_deleted": True}
SP_OPTS = cdb.SparseSearchOptions(0, None, True, 5)
KIND_SOURCES = pm.KIND_SOURCES


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def check(got, want):
    assert np.array_equal(got[2], want[2])
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(bits(got[1]), bits(want[1]))


def csr_rows(c):
    o, d, v = c
    return [list(zip(d[int(o[i]):int(o[i + 1])].tolist(), v[int(o[i]):int(o[i + 1])].tolist())) for i in range(len(o) - 1)]


class Corpus:
    """N rows in every kind of index over one id space, with deletes; per-query inputs for BMAX queries"""

    def __init__(self, seed=31):
        rng = np.random.default_rng(seed)
        centres = rng.normal(size=(64, DIM)).astype(np.float32)
        self.vecs = (centres[rng.integers(0, 64, N)] + 0.4 * rng.normal(size=(N, DIM))).astype(np.float32)
        self.vecs /= np.abs(self.vecs).max() * 1.01
        self.sp_corpus = zipf_csr(41, N, vocab=VOCAB, mean_pairs=24)
        self.tf_corpus = zipf_docs(42, N, vocab=VOCAB, mean_terms=16)
        self.dead = rng.choice(N, 300, replace=False)
        self.dq = (self.vecs[rng.integers(0, N, BMAX)] + 0.05 * rng.normal(size=(BMAX, DIM))).astype(np.float32)
        self.sq = csr_rows(zipf_csr(43, BMAX, vocab=VOCAB, mean_pairs=10))
        self.tq = zipf_queries(44, BMAX, vocab=VOCAB)

    def indexes(self, r0=0, r1=N, device=0, hnsw_base=None):
        """-> dict of the four kinds of index over rows [r0, r1)"""
        hn = cdb.DenseIndex(dim=DIM, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=r1 - r0 + 1, keep_raw_f32=True,
                            id_base=r0 if hnsw_base is None else hnsw_base, device=device)
        hn.append(self.vecs[r0:r1])
        hn.build_graph(num_levels=4, neighbors_count=16, level0_neighbors_count=32, ef_construction=64, shortlist_size=32)
        raw = cdb.DenseIndex(dim=DIM, capacity=r1 - r0, tensor_prefilter=True, id_base=r0, device=device)
        raw.append(self.vecs[r0:r1])
        part = slice_csr(self.sp_corpus, r0, r1)
        sp = cdb.SparseIndex(capacity_rows=r1 - r0, capacity_pairs=len(part[1]) + 8, id_base=r0, device=device)
        sp.append(part)
        part = slice_csr(self.tf_corpus, r0, r1)
        tf = cdb.TfIdfIndex(capacity_rows=r1 - r0, capacity_pairs=len(part[1]) + 8, id_base=r0, device=device)
        tf.append(part, 1)
        mine = self.dead[(self.dead >= r0) & (self.dead < r1)] - r0
        raw.delete_rows(mine)
        sp.delete_embedding(mine)
        tf.delete_embedding(mine, 2)
        return {"hn": hn, "raw": raw, "sp": sp, "tf": tf}

    def inputs(self, b, off=0):
        return self.dq[off:off + b], self.sq[off:off + b], self.tq[off:off + b]


def kinds_of(case, b, seed=0):
    rng = np.random.default_rng(seed + b)
    if case in ("0", "1", "2"):
        return np.full(b, int(case), np.uint8)
    if case == "02":
        return rng.choice([0, 2], b).astype(np.uint8)
    if case == "01":
        return rng.choice([0, 1], b).astype(np.uint8)
    k = np.arange(b) % 3
    rng.shuffle(k)
    return k.astype(np.uint8)


def assemble(kinds, per_kind):
    """rows of per-kind results (ids, scores, counts, err over that kind's queries) back in request order"""
    kinds = np.asarray(kinds)
    out = None
    for kind, r in per_kind.items():
        rows = np.flatnonzero(kinds == kind)
        if out is None:
            out = [np.zeros((len(kinds),) + x.shape[1:], x.dtype) for x in r]
        for o, x in zip(out, r):
            o[rows] = x
    return tuple(out)


def sub_lists(kinds, dq, sq, tq, run):
    """each source's own search of its batch (the queries whose kind names it, in request order) -> {source: (ids, counts)}
    and the dense error bytes of that batch"""
    _, batches = cdb.split_mixed(kinds, dq, sq, tq)
    out, err = {}, None
    for name, q in batches.items():
        r = run[name](q)
        out[name] = (r[0], r[2])
        if name == "dense":
            err = r[3]
    return out, err


def check_err(kinds, got_err, dense_err):
    """error bytes: the dense search's at the queries that name dense, 0 at sparse + TF-IDF queries"""
    dense_rows = np.flatnonzero(np.isin(kinds, (0, 1)))
    assert np.array_equal(got_err[dense_rows], dense_err)
    assert not got_err[np.asarray(kinds) == 2].any()


# ---------------------------------------------------------------- single index
@pytest.fixture(scope="module")
def single():
    c = Corpus()
    ix = c.indexes()
    yield c, ix
    for h in ix.values():
        h.close()


CASES = [("0", 64, 10), ("1", 64, 10), ("2", 64, 341), ("02", 64, 10), ("01", 257, 21), ("012", 1, 10), ("012", 64, 1),
         ("012", 1024, 10), ("012", 300, 341)]


def single_split(ix, dense_key, dense_opts, kinds, dq, sq, tq, top_k):
    handles = {"dense": ix[dense_key], "sparse": ix["sp"], "tfidf": ix["tf"]}
    opts = {"dense": dense_opts, "sparse": SP_OPTS, "tfidf": None}
    qs = {"dense": dq, "sparse": sq, "tfidf": tq}
    per_kind = {}
    for kind in np.unique(kinds).tolist():
        rows = np.flatnonzero(kinds == kind)
        kw = {n: (handles[n], [qs[n][i] for i in rows] if n != "dense" else dq[rows], opts[n]) for n in KIND_SOURCES[kind]}
        kw = {n: v if n != "tfidf" else v[:2] for n, v in kw.items()}
        per_kind[kind] = cdb.hybrid_batch_search(top_k, 60.0, **kw)
    return assemble(kinds, per_kind)


def single_run(ix, dense_key, dense_opts, top_k):
    k3 = 3 * top_k
    return {"dense": lambda q: ix[dense_key].batch_search(q, k3, **dense_opts),
            "sparse": lambda q: ix["sp"].batch_search(q, cdb.SparseSearchOptions(k3, None, True, 5)),
            "tfidf": lambda q: ix["tf"].batch_search(q, k3)}


@pytest.mark.parametrize("dense_key", ["hn", "raw"])
@pytest.mark.parametrize("case,b,top_k", CASES, ids=lambda x: str(x))
def test_single_index_mixed_equals_the_split_by_kind(single, dense_key, case, b, top_k):
    c, ix = single
    dense_opts = DENSE_HNSW if dense_key == "hn" else DENSE_TC
    kinds = kinds_of(case, b)
    dq, sq, tq = c.inputs(b)
    got = cdb.hybrid_batch_search_mixed(kinds, top_k, 60.0, dense=(ix[dense_key], dq, dense_opts), sparse=(ix["sp"], sq, SP_OPTS),
                                        tfidf=(ix["tf"], tq))
    assert got[0].shape == (b, 6 * top_k)
    want = single_split(ix, dense_key, dense_opts, kinds, dq, sq, tq, top_k)
    check(got, want)
    assert np.array_equal(got[3], want[3])
    lists, dense_err = sub_lists(kinds, dq, sq, tq, single_run(ix, dense_key, dense_opts, top_k))
    check(got, pm.fuse_mixed(kinds, lists, 60.0, ld_out=6 * top_k))
    if dense_err is not None:
        check_err(kinds, got[3], dense_err)


def test_error_bytes_land_at_the_dense_queries():
    """a u8 cosine index with all-zero rows: every dense search sets CDB_ERRFLAG_CALCULATION (cosine.rs:230-231), so the
    error bytes of a shuffled batch are 1 exactly where the query names dense, on the single index and a one-slot group"""
    c = Corpus(seed=35)
    vecs = c.vecs.copy()
    vecs[[7, 9000]] = -1.0
    kw = dict(storage_type=cdb.StorageType.UnsignedByte, metric=cdb.DistanceMetricKind.Cosine)
    ix = cdb.DenseIndex(dim=DIM, capacity=N, **kw)
    ix.append(vecs)
    sp = cdb.SparseIndex(capacity_rows=N, capacity_pairs=len(c.sp_corpus[1]))
    sp.append(c.sp_corpus)
    tf = cdb.TfIdfIndex(capacity_rows=N, capacity_pairs=len(c.tf_corpus[1]))
    tf.append(c.tf_corpus, 1)
    g = ShardGroup.local([0])
    g.attach(0, ix)
    g.attach_sparse(0, sp)
    g.attach_tfidf(0, tf)
    opts = {"mode": cdb.SearchMode.BRUTE_CODES}
    for b in (1, 64, 200):
        kinds = kinds_of("012", b, seed=4)
        dq, sq, tq = c.inputs(b)
        names_dense = np.isin(kinds, (0, 1)).astype(np.uint8)
        got = cdb.hybrid_batch_search_mixed(kinds, 10, 60.0, dense=(ix, dq, opts), sparse=(sp, sq, SP_OPTS), tfidf=(tf, tq))
        want = single_split({"raw": ix, "sp": sp, "tf": tf}, "raw", opts, kinds, dq, sq, tq, 10)
        check(got, want)
        assert np.array_equal(got[3], want[3]) and np.array_equal(got[3], names_dense)
        got = g.hybrid_search_mixed(kinds, 10, 60.0, dense=(dq, opts), sparse=(sq, SP_OPTS), tfidf=tq)
        want = group_split(g, opts, kinds, dq, sq, tq, 10)
        check(got, want)
        assert np.array_equal(got[3], want[3]) and np.array_equal(got[3], names_dense)
    g.close(); ix.close(); sp.close(); tf.close()


def test_single_index_searches_each_source_once(single):
    c, ix = single
    b, top_k = 96, 10
    kinds = kinds_of("012", b, seed=3)
    dq, sq, tq = c.inputs(b)
    run = single_run(ix, "hn", DENSE_HNSW, top_k)
    _, batches = cdb.split_mixed(kinds, dq, sq, tq)
    sub = 0
    for name, q in batches.items():
        n0 = cdb.kernel_launch_count()
        run[name](q)
        sub += cdb.kernel_launch_count() - n0
    kw = dict(dense=(ix["hn"], dq, DENSE_HNSW), sparse=(ix["sp"], sq, SP_OPTS), tfidf=(ix["tf"], tq))
    n0 = cdb.kernel_launch_count()
    cdb.hybrid_batch_search_mixed(kinds, top_k, 60.0, **kw)
    mixed = cdb.kernel_launch_count() - n0
    assert mixed == sub + 3                                     # the three sub-searches and one fusion per kind
    n0 = cdb.kernel_launch_count()
    single_split(ix, "hn", DENSE_HNSW, kinds, dq, sq, tq, top_k)
    assert cdb.kernel_launch_count() - n0 > mixed              # the split searches every source twice
    n0 = cdb.kernel_launch_count()
    got = cdb.hybrid_batch_search_mixed(kinds, 0, 60.0, **kw)
    assert cdb.kernel_launch_count() == n0 and not got[2].any()


def torch_of(a, dev):
    import torch
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(a.dtype, a.dtype)
    return torch.from_numpy(a.view(view)).to(dev)


@pytest.mark.parametrize("case,b", [("012", 200), ("2", 33), ("01", 1)])
def test_single_index_device_form_on_a_side_stream(single, case, b):
    import ctypes as C
    import torch
    from cosdata_b200 import _lib
    from cosdata_b200.api import _query_csr, sparse_csr
    c, ix = single
    dev, top_k = torch.device("cuda", 0), 10
    kinds = kinds_of(case, b, seed=9)
    dq, sq, tq = c.inputs(b, off=100)
    host = cdb.hybrid_batch_search_mixed(kinds, top_k, 60.0, dense=(ix["raw"], dq, DENSE_TC), sparse=(ix["sp"], sq, SP_OPTS),
                                         tfidf=(ix["tf"], tq))
    _, batches = cdb.split_mixed(kinds, dq, sq, tq)
    src, alive = _lib.HybridMixedSources(), [kinds]
    src.kinds = kinds.ctypes.data
    src.dense, src.dense_params = ix["raw"]._h, ix["raw"].params(0, **DENSE_TC)
    src.sparse, src.sparse_params = ix["sp"].h, SP_OPTS.params()
    src.tfidf = ix["tf"].h
    if "dense" in batches:
        t = torch_of(batches["dense"], dev)
        src.n_dense, src.dense_queries = t.shape[0], t.data_ptr()
        alive.append(t)
    if "sparse" in batches:
        ts = [torch_of(a, dev) for a in sparse_csr(batches["sparse"])]
        src.n_sparse = ts[0].numel() - 1
        src.sparse_offsets, src.sparse_dims, src.sparse_values = (t.data_ptr() for t in ts)
        alive += ts
    if "tfidf" in batches:
        tt = [torch_of(a, dev) for a in _query_csr(batches["tfidf"])]
        src.n_tfidf = tt[0].numel() - 1
        src.tfidf_offsets, src.tfidf_hashes = (t.data_ptr() for t in tt)
        alive += tt
    ids = torch.zeros((b, 6 * top_k), dtype=torch.int32, device=dev)
    sc = torch.zeros((b, 6 * top_k), dtype=torch.float32, device=dev)
    cnt = torch.zeros(b, dtype=torch.int32, device=dev)
    err = torch.full((b,), 0xEE, dtype=torch.uint8, device=dev)
    s = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    assert _lib.load().cdb_hybrid_search_batch_mixed_device(C.byref(src), b, top_k, 60.0, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                                                            err.data_ptr(), C.c_void_p(s.cuda_stream)) == 0
    s.synchronize()
    check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), host)
    assert np.array_equal(err.cpu().numpy(), host[3])


# ---------------------------------------------------------------- shard groups
@pytest.fixture(scope="module")
def grouped():
    """a 2-slot loopback group of each dense kind (HNSW shards spaced 1 << 20 apart, f32 shards) sharing the text shards"""
    c = Corpus(seed=33)
    bounds = [shard_range(N, 2, r)[0] for r in range(2)] + [N]
    gh, gr = ShardGroup.local([0, 0]), ShardGroup.local([0, 0])
    parts = []
    for r in range(2):
        ix = c.indexes(bounds[r], bounds[r + 1], hnsw_base=r << 20)
        gh.attach(r, ix["hn"])
        gr.attach(r, ix["raw"])
        for g in (gh, gr):
            g.attach_sparse(r, ix["sp"])
            g.attach_tfidf(r, ix["tf"])
        parts.append(ix)
    yield c, {"hn": gh, "raw": gr}
    gh.close(); gr.close()
    for ix in parts:
        for h in ix.values():
            h.close()


def group_split(g, dense_opts, kinds, dq, sq, tq, top_k, stride=1):
    qs = {"dense": dq, "sparse": sq, "tfidf": tq}
    per_kind = {}
    for kind in np.unique(kinds).tolist():
        rows = np.flatnonzero(kinds == kind)
        kw = {}
        for n in KIND_SOURCES[kind]:
            q = dq[rows] if n == "dense" else [qs[n][i] for i in rows]
            kw[n] = q if n == "tfidf" else (q, dense_opts if n == "dense" else SP_OPTS)
        per_kind[kind] = g.hybrid_search(top_k, 60.0, dense_id_stride=stride, **kw)
    return assemble(kinds, per_kind)


def group_run(g, dense_opts, top_k, md=False):
    k3 = 3 * top_k
    dense = ((lambda q: g.search_filtered(q, [None] * len(q), k3, **{k: v for k, v in dense_opts.items() if k != "mode"})) if md
             else (lambda q: g.search(q, k3, **dense_opts)))
    return {"dense": dense, "sparse": lambda q: g.search_sparse(q, cdb.SparseSearchOptions(k3, None, True, 5)),
            "tfidf": lambda q: g.search_tfidf(q, k3)}


@pytest.mark.parametrize("dense_key", ["hn", "raw"])
@pytest.mark.parametrize("case,b,top_k", [("0", 64, 10), ("2", 64, 10), ("02", 64, 341), ("012", 1, 10), ("012", 1024, 10),
                                          ("012", 200, 341)], ids=lambda x: str(x))
def test_group_mixed_equals_the_split_by_kind(grouped, dense_key, case, b, top_k):
    c, groups = grouped
    g = groups[dense_key]
    dense_opts = DENSE_HNSW if dense_key == "hn" else DENSE_TC
    kinds = kinds_of(case, b, seed=1)
    dq, sq, tq = c.inputs(b)
    got = g.hybrid_search_mixed(kinds, top_k, 60.0, dense=(dq, dense_opts), sparse=(sq, SP_OPTS), tfidf=tq)
    want = group_split(g, dense_opts, kinds, dq, sq, tq, top_k)
    check(got, want)
    assert np.array_equal(got[3], want[3])
    lists, dense_err = sub_lists(kinds, dq, sq, tq, group_run(g, dense_opts, top_k))
    check(got, pm.fuse_mixed(kinds, lists, 60.0, ld_out=6 * top_k))
    if dense_err is not None:
        check_err(kinds, got[3], dense_err)
    if case == "012":
        n0 = cdb.kernel_launch_count()
        g.hybrid_search_mixed(kinds, top_k, 60.0, dense=(dq, dense_opts), sparse=(sq, SP_OPTS), tfidf=tq)
        mixed = cdb.kernel_launch_count() - n0
        run, (_, batches) = group_run(g, dense_opts, top_k), cdb.split_mixed(kinds, dq, sq, tq)
        n0 = cdb.kernel_launch_count()
        for name, q in batches.items():
            run[name](q)
        assert mixed == cdb.kernel_launch_count() - n0 + len(np.unique(kinds))


def test_group_batch_above_one_fusion_chunk(grouped):
    """sparse + TF-IDF and dense + sparse queries at top_k 341: a chunk holds 256 MB / ((1023 + 1023) * 8 + 9) request
    positions (the widest kind, and the dense error byte), 16,391, so a batch 40 larger takes two, each a contiguous
    range of every source's batch; a sample on both sides of the boundary against both oracles"""
    c, groups = grouped
    g, top_k = groups["raw"], 341
    chunk = (256 << 20) // ((3 * top_k + 3 * top_k) * 8 + 9)
    b = chunk + 40
    rng = np.random.default_rng(12)
    kinds = rng.choice([0, 2], b).astype(np.uint8)
    dq = (c.vecs[rng.integers(0, N, b)] + 0.05 * rng.normal(size=(b, DIM))).astype(np.float32)
    sq = csr_rows(zipf_csr(45, b, vocab=VOCAB, mean_pairs=10))
    tq = zipf_queries(46, b, vocab=VOCAB)
    got = g.hybrid_search_mixed(kinds, top_k, 60.0, dense=(dq, DENSE_TC), sparse=(sq, SP_OPTS), tfidf=tq)
    rows = np.unique(np.concatenate([np.arange(8), np.arange(chunk - 8, chunk + 8), np.arange(b - 8, b), rng.choice(b, 40)]))
    lists, _ = sub_lists(kinds, dq, sq, tq, group_run(g, DENSE_TC, top_k))
    # fuse_mixed over the sample alone: its queries in request order with their rows of each source's lists
    mapping, _ = pm.query_mapping(kinds)
    pick = {"dense": [], "sparse": [], "tfidf": []}
    for q in rows:
        _, i1, i2, kind = mapping[q]
        pick[KIND_SOURCES[kind][0]].append(i1)
        pick[KIND_SOURCES[kind][1]].append(i2)
    sub = {n: (lists[n][0][idx], lists[n][1][idx]) for n, idx in pick.items() if idx}
    check(tuple(x[rows] for x in got[:3]), pm.fuse_mixed(kinds[rows], sub, 60.0, ld_out=6 * top_k))
    split = group_split(g, DENSE_TC, kinds[rows], dq[rows], [sq[i] for i in rows], [tq[i] for i in rows], top_k)
    check(tuple(x[rows] for x in got[:3]), split)
    assert np.array_equal(got[3][rows], split[3])


def test_group_device_form_with_a_tfidf_source_matches_the_host_form(grouped):
    import torch
    from cosdata_b200.api import _query_csr, sparse_csr
    c, _ = grouped
    dev, top_k = torch.device("cuda", 0), 10
    one = c.indexes()
    s = torch.cuda.Stream(dev)
    for g in (ShardGroup.rank(None, 1, 0, 0), ShardGroup.local([0])):
        g.attach(0, one["raw"])
        g.attach_sparse(0, one["sp"])
        g.attach_tfidf(0, one["tf"])
        for case, b in (("012", 256), ("2", 40), ("1", 1)):
            kinds = kinds_of(case, b, seed=5)
            dq, sq, tq = c.inputs(b, off=200)
            host = g.hybrid_search_mixed(kinds, top_k, 60.0, dense=(dq, DENSE_TC), sparse=(sq, SP_OPTS), tfidf=tq)
            _, batches = cdb.split_mixed(kinds, dq, sq, tq)
            alive, kw = [], {}
            if "dense" in batches:
                t = torch_of(batches["dense"], dev)
                kw["dense"] = (t.data_ptr(), DENSE_TC)
                alive.append(t)
            if "sparse" in batches:
                ts = [torch_of(a, dev) for a in sparse_csr(batches["sparse"])]
                kw["sparse"] = (tuple(t.data_ptr() for t in ts), SP_OPTS)
                alive += ts
            if "tfidf" in batches:
                o, h = _query_csr(batches["tfidf"])
                tt = [torch_of(o, dev), torch_of(h, dev)]
                kw["tfidf"] = (tt[0].data_ptr(), tt[1].data_ptr(), int(o[-1]))
                alive += tt
            ids = torch.zeros((b, 6 * top_k), dtype=torch.int32, device=dev)
            sc = torch.zeros((b, 6 * top_k), dtype=torch.float32, device=dev)
            cnt = torch.zeros(b, dtype=torch.int32, device=dev)
            err = torch.full((b,), 0xEE, dtype=torch.uint8, device=dev)
            torch.cuda.synchronize(dev)
            g.hybrid_search_mixed_device(kinds, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), err.data_ptr(), s.cuda_stream, top_k, 60.0,
                                         **kw)
            s.synchronize()
            check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), host)
            assert np.array_equal(err.cpu().numpy(), host[3])
        g.close()
    for h in one.values():
        h.close()


def test_one_slot_group_over_a_replica_graph():
    from tests.test_gpu_sharded_hybrid import REPLICAS, replica_index
    vecs, ix, sp = replica_index()
    tf_corpus = zipf_docs(53, REPLICAS * 2000, vocab=500, mean_terms=8)
    tf = cdb.TfIdfIndex(capacity_rows=REPLICAS * 2000, capacity_pairs=len(tf_corpus[1]))
    tf.append(tf_corpus, 1)
    g = ShardGroup.local([0])
    g.attach(0, ix)
    g.attach_sparse(0, sp)
    g.attach_tfidf(0, tf)
    rng = np.random.default_rng(5)
    b = 90
    kinds = kinds_of("012", b, seed=8)
    dq = (vecs[rng.integers(0, vecs.shape[0], b)] + 0.02 * rng.normal(size=(b, 32))).astype(np.float32)
    sq = csr_rows(zipf_csr(52, b, vocab=500, mean_pairs=6))
    tq = zipf_queries(54, b, vocab=500)
    dense_opts = {"mode": cdb.SearchMode.HNSW, "ef_search": 64, "shortlist_size": 64}
    for top_k in (1, 10, 341):
        got = g.hybrid_search_mixed(kinds, top_k, 60.0, dense=(dq, dense_opts), sparse=(sq, SP_OPTS), tfidf=tq, dense_id_stride=REPLICAS)
        want = group_split(g, dense_opts, kinds, dq, sq, tq, top_k, stride=REPLICAS)
        check(got, want)
        assert np.array_equal(got[3], want[3])
        lists, dense_err = sub_lists(kinds, dq, sq, tq, group_run(g, dense_opts, top_k, md=True))
        check(got, pm.fuse_mixed(kinds, lists, 60.0, dense_stride=REPLICAS, ld_out=6 * top_k))
        check_err(kinds, got[3], dense_err)
    g.close(); ix.close(); sp.close(); tf.close()
