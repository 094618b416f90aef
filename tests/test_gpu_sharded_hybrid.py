"""Hybrid search over a shard group (cdb_hybrid_search_batch_sharded[_device]) against tests/pyhybrid.py, bit for bit on
ids, counts and score bits:
  * composition: every pairing on groups of 2 and 3 shards, batch 1, 64 and 1024, top_k 1, 10 and 341, equals the fusion of
    the group's own sub-searches at k = 3 * top_k (HNSW and BRUTE_RAW dense, sparse with and without re-rank and with a
    threshold), before and after deletes in every kind of shard;
  * whole corpus: where every sub-search is exact across shards (BRUTE_RAW on the tensor-core path, sparse, TF-IDF), equal
    to cdb_hybrid_search_batch over single indexes holding the whole corpus, also over two fusion chunks with a TF-IDF source;
  * replica graphs: a one-slot group over a replica-graph index (the hybrid search cdb_hybrid_search_batch refuses), a
    two-shard replica group, and the refusal of a group that mixes replica and plain graphs;
  * the device form on a side stream equals the host form, on a per-rank group and a one-device local group; a TF-IDF
    source is refused there; error bytes are written only with a dense source; top_k = 0 launches nothing.
One GPU: the shards share device 0 and the gathers are the copy-based loopback; with >= 2 GPUs the same checks run over
NCCL."""
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from cosdata_b200.sharding import ShardGroup, shard_range
from tests import pyhybrid as ph
from tests.sparse_data import slice_csr, zipf_csr
from tests.tfidf_data import zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu
N, DIM, BMAX, VOCAB = 20_000, 64, 1024, 3000
DENSE_HNSW = {"mode": cdb.SearchMode.HNSW, "ef_search": 256, "shortlist_size": 64}
DENSE_TC = {"mode": cdb.SearchMode.BRUTE_RAW, "tensor_with_deleted": True}
PAIRS = [("dense", "sparse"), ("dense", "tfidf"), ("sparse", "tfidf")]
HN_GAP = 1 << 20


def devices(n):
    return list(range(n)) if cdb.device_count() >= n else [0] * n


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def check(got, want):
    ids, scores, counts = got[:3]
    w_ids, w_scores, w_counts = want[:3]
    assert np.array_equal(counts, w_counts)
    assert np.array_equal(ids, w_ids)
    assert np.array_equal(bits(scores), bits(w_scores))


class World:
    """N rows split over `nshards` shards of every kind at the same global id ranges, next to whole-corpus indexes; two
    groups share the text shards: `gh` with HNSW dense shards (graphs built on the GPU), `gr` with f32 shards for the
    tensor-core brute force.  Deletes go to every shard and whole index that holds the row."""

    def __init__(self, nshards, seed=31):
        rng = np.random.default_rng(seed + nshards)
        centres = rng.normal(size=(64, DIM)).astype(np.float32)
        vecs = (centres[rng.integers(0, 64, N)] + 0.4 * rng.normal(size=(N, DIM))).astype(np.float32)
        vecs /= np.abs(vecs).max() * 1.01
        sp_corpus = zipf_csr(41, N, vocab=VOCAB, mean_pairs=24)
        tf_corpus = zipf_docs(42, N, vocab=VOCAB, mean_terms=16)
        self.bounds = [shard_range(N, nshards, r)[0] for r in range(nshards)] + [N]
        devs = devices(nshards)
        self.gh, self.gr = ShardGroup.local(devs), ShardGroup.local(devs)
        self.hn, self.raw, self.sp, self.tf = [], [], [], []
        for r in range(nshards):
            b0, b1 = self.bounds[r], self.bounds[r + 1]
            # a graph build keeps one more row for its root, so the HNSW shards' id ranges are spaced HN_GAP apart
            hn = cdb.DenseIndex(dim=DIM, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=b1 - b0 + 1, keep_raw_f32=True,
                                id_base=r * HN_GAP, device=devs[r])
            hn.append(vecs[b0:b1])
            hn.build_graph(num_levels=4, neighbors_count=16, level0_neighbors_count=32, ef_construction=64, shortlist_size=32)
            raw = cdb.DenseIndex(dim=DIM, capacity=b1 - b0, tensor_prefilter=True, id_base=b0, device=devs[r])
            raw.append(vecs[b0:b1])
            part = slice_csr(sp_corpus, b0, b1)
            sp = cdb.SparseIndex(capacity_rows=b1 - b0, capacity_pairs=len(part[1]) + 8, id_base=b0, device=devs[r])
            sp.append(part)
            part = slice_csr(tf_corpus, b0, b1)
            tf = cdb.TfIdfIndex(capacity_rows=b1 - b0, capacity_pairs=len(part[1]) + 8, id_base=b0, device=devs[r])
            tf.append(part, 1)
            self.gh.attach(r, hn)
            self.gr.attach(r, raw)
            for g in (self.gh, self.gr):
                g.attach_sparse(r, sp)
                g.attach_tfidf(r, tf)
            self.hn.append(hn); self.raw.append(raw); self.sp.append(sp); self.tf.append(tf)
        self.w_raw = cdb.DenseIndex(dim=DIM, capacity=N, tensor_prefilter=True)
        self.w_raw.append(vecs)
        self.w_sp = cdb.SparseIndex(capacity_rows=N, capacity_pairs=len(sp_corpus[1]))
        self.w_sp.append(sp_corpus)
        self.w_tf = cdb.TfIdfIndex(capacity_rows=N, capacity_pairs=len(tf_corpus[1]))
        self.w_tf.append(tf_corpus, 1)
        self.dq = (vecs[rng.integers(0, N, BMAX)] + 0.05 * rng.normal(size=(BMAX, DIM))).astype(np.float32)
        self.sq = zipf_csr(43, BMAX, vocab=VOCAB, mean_pairs=10)
        self.tq = zipf_queries(44, BMAX, vocab=VOCAB)
        self.version = 1

    def delete(self, rows):
        """global rows out of every kind of shard (and the whole indexes)"""
        rows = np.unique(np.asarray(rows, np.uint32))
        self.version += 1
        for r in range(len(self.hn)):
            mine = rows[(rows >= self.bounds[r]) & (rows < self.bounds[r + 1])] - self.bounds[r]
            assert mine.size
            self.hn[r].delete_rows(mine)
            self.raw[r].delete_rows(mine)
            self.sp[r].delete_embedding(mine)
            self.tf[r].delete_embedding(mine, self.version)
        self.w_raw.delete_rows(rows)
        self.w_sp.delete_embedding(rows)
        self.w_tf.delete_embedding(rows, self.version)

    def queries(self, b):
        return self.dq[:b], slice_csr(self.sq, 0, b), self.tq[:b]

    def close(self):
        self.gh.close(); self.gr.close()
        for x in self.hn + self.raw + self.sp + self.tf + [self.w_raw, self.w_sp, self.w_tf]:
            x.close()


@pytest.fixture(scope="module", params=[2, 3], ids=lambda n: f"{n}shards")
def world(request):
    w = World(request.param)
    w.delete(np.random.default_rng(request.param).choice(N, 400, replace=False))
    yield w
    w.close()


def group_sources(g, pair, dq, sq, tq, dense_opts, sp_opts, md=False):
    """-> (hybrid_search keywords, function top_k -> the group's own two lists (ids, scores, counts) at 3 * top_k)"""
    kw, run = {}, {}
    if "dense" in pair:
        kw["dense"] = (dq, dense_opts)
        if md:
            run["dense"] = lambda k3: g.search_filtered(dq, [None] * len(dq), k3, **{k: v for k, v in dense_opts.items() if k != "mode"})[:3]
        else:
            run["dense"] = lambda k3: g.search(dq, k3, **dense_opts)[:3]
    if "sparse" in pair:
        kw["sparse"] = (sq, sp_opts)
        run["sparse"] = lambda k3: g.search_sparse(sq, cdb.SparseSearchOptions(k3, sp_opts.early_terminate_threshold, sp_opts.rerank,
                                                                                sp_opts.reranking_factor))
    if "tfidf" in pair:
        kw["tfidf"] = tq
        run["tfidf"] = lambda k3: g.search_tfidf(tq, k3)
    return kw, lambda top_k: (run[pair[0]](3 * top_k), run[pair[1]](3 * top_k))


def expected(lists, top_k, strides=(1, 1), k=60.0):
    (a, _, ca), (b, _, cb) = lists
    return ph.fuse_batch(a, ca, b, cb, k, strides, ld_out=6 * top_k)


SPARSE_OPTS = [cdb.SparseSearchOptions(0, 0.0, False, 5), cdb.SparseSearchOptions(0, 0.5, False, 5),
               cdb.SparseSearchOptions(0, 0.0, True, 5)]
CASES = [(1, 1), (1, 341), (64, 10), (64, 341), (1024, 10), (1024, 1)]


def compose(w, pair, cases):
    i = 0
    for dense_opts, g in ((DENSE_HNSW, w.gh), (DENSE_TC, w.gr)) if "dense" in pair else ((None, w.gh),):
        for b, top_k in cases:
            sp_opts = SPARSE_OPTS[i % len(SPARSE_OPTS)]
            i += 1
            kw, lists = group_sources(g, pair, *w.queries(b), dense_opts, sp_opts)
            got = g.hybrid_search(top_k, 60.0, **kw)
            assert got[0].shape == (b, 6 * top_k)
            check(got, expected(lists(top_k), top_k))
            if "dense" in pair:
                assert np.array_equal(got[3], g.search(w.dq[:b], 3 * top_k, **dense_opts)[3])
            else:
                assert not got[3].any()


@pytest.mark.parametrize("pair", PAIRS, ids="-".join)
def test_group_hybrid_equals_the_fusion_of_the_group_searches(world, pair):
    compose(world, pair, CASES)


def test_composition_after_more_deletes(world):
    """the first-ranked rows of some queries go, in every kind of shard"""
    top = [world.gr.search(world.dq[:8], 1, **DENSE_TC)[0][:, 0], world.gh.search_sparse(world.queries(8)[1], cdb.SparseSearchOptions(1))[0][:, 0],
           world.gh.search_tfidf(world.tq[:8], 1)[0][:, 0]]
    extra = np.concatenate([t[t != cdb.INVALID_ID] for t in top] + [np.random.default_rng(7).choice(N, 200, replace=False)])
    world.delete(np.setdiff1d(extra, np.flatnonzero(world.w_raw.deleted_rows())))
    for pair in PAIRS:
        compose(world, pair, [(64, 10), (1, 341)])


@pytest.mark.parametrize("pair", PAIRS, ids="-".join)
def test_group_hybrid_equals_whole_corpus_hybrid(world, pair):
    for b, top_k, sp_opts in ((1024, 10, SPARSE_OPTS[0]), (64, 341, SPARSE_OPTS[2]), (1024, 341, SPARSE_OPTS[1])):
        dq, sq, tq = world.queries(b)
        kw, _ = group_sources(world.gr, pair, dq, sq, tq, DENSE_TC, sp_opts)
        got = world.gr.hybrid_search(top_k, 60.0, **kw)
        whole = {"dense": (world.w_raw, dq, DENSE_TC), "sparse": (world.w_sp, sq, sp_opts), "tfidf": (world.w_tf, tq)}
        want = cdb.hybrid_batch_search(top_k, 60.0, **{p: whole[p] for p in pair})
        check(got, want)
        assert np.array_equal(got[3], want[3])


def test_tfidf_source_over_two_fusion_chunks(world):
    """sparse + TF-IDF at top_k 341: a fusion chunk holds 256 MB / ((1023 + 512) * 8 + 8) bytes of lists, 21845 queries, so
    a batch of five more takes two.  The group's idf is computed once for the whole batch and each chunk scores its window
    of the TF-IDF query CSR.  Every query against the whole-corpus hybrid; the fusion of the group's own searches on a sample
    that holds both sides of the chunk boundary."""
    top_k = 341
    chunk = (256 << 20) // ((3 * top_k + min(3 * top_k, 512)) * 8 + 8)
    b = chunk + 5
    sq, tq = zipf_csr(45, b, vocab=VOCAB, mean_pairs=10), zipf_queries(46, b, vocab=VOCAB)
    sp_opts = SPARSE_OPTS[2]
    kw, lists = group_sources(world.gh, ("sparse", "tfidf"), None, sq, tq, None, sp_opts)
    got = world.gh.hybrid_search(top_k, 60.0, **kw)
    check(got, cdb.hybrid_batch_search(top_k, 60.0, sparse=(world.w_sp, sq, sp_opts), tfidf=(world.w_tf, tq)))
    (a, _, ca), (b_ids, _, cb) = lists(top_k)
    rows = np.unique(np.concatenate([np.arange(8), np.arange(chunk - 8, b), np.random.default_rng(3).choice(b, 48)]))
    check(tuple(x[rows] for x in got[:3]), ph.fuse_batch(a[rows], ca[rows], b_ids[rows], cb[rows], 60.0, ld_out=6 * top_k))


def test_error_bytes_only_with_a_dense_source_and_top_k_zero(world):
    L = _lib.load()
    dq, sq, tq = world.queries(64)
    for pair in PAIRS:
        kw, _ = group_sources(world.gr, pair, dq, sq, tq, DENSE_TC, SPARSE_OPTS[0])
        src, keep, nq = world.gr._hybrid_sources(kw.get("dense"), kw.get("sparse"), kw.get("tfidf"), 1, True)
        ids, sc = np.zeros((64, 60), np.uint32), np.zeros((64, 60), np.float32)
        cnt, err = np.zeros(64, np.uint32), np.full(64, 0xEE, np.uint8)
        assert L.cdb_hybrid_search_batch_sharded(world.gr._h, C.byref(src), 64, 10, 60.0, ids.ctypes.data, sc.ctypes.data, cnt.ctypes.data,
                                                 err.ctypes.data) == 0
        if "dense" in pair:
            assert np.array_equal(err, world.gr.search(dq, 30, **DENSE_TC)[3])
        else:
            assert (err == 0xEE).all()
        n0 = cdb.kernel_launch_count()
        ids, _, counts, _ = world.gr.hybrid_search(0, 60.0, **kw)
        assert cdb.kernel_launch_count() == n0 and ids.shape == (64, 0) and not counts.any()


def test_slot_without_a_shard_of_a_named_kind():
    devs = devices(2)
    g = ShardGroup.local(devs)
    ixs = []
    for r in range(2):
        ix = cdb.DenseIndex(dim=8, capacity=10, id_base=10 * r, device=devs[r])
        ix.append(np.ones((10, 8), np.float32))
        g.attach(r, ix)
        ixs.append(ix)
    sp = cdb.SparseIndex(capacity_rows=10, capacity_pairs=10, device=devs[0])
    g.attach_sparse(0, sp)
    with pytest.raises(cdb.CosdataError) as e:
        g.hybrid_search(10, 60.0, dense=(np.ones((2, 8), np.float32), None), sparse=([[(0, 1.0)]] * 2, None))
    assert e.value.status == cdb.Status.INVALID_PARAMS and "sparse shard" in str(e.value)
    g.close()
    for x in ixs + [sp]:
        x.close()


# ---------------------------------------------------------------- replica graphs
REPLICAS = 4


def replica_index(seed=7, n=2000, id_base=0):
    """a replica graph of mdgraph.replica_population (ids i * 4 + j) and a sparse index over its id space"""
    from tests import mdgraph
    pop = mdgraph.replica_population(n=n, dim=32, md_dims=6, levels=4, seed=seed)
    vecs = pop["vecs"]
    ix = cdb.DenseIndex(dim=32, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=vecs.shape[0] + 2, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph_replicas(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], pop["md_bits"],
                            pop["md_mags"], pop["main_root_md"], pop["pseudo_root_md"], 4, 16, 32, 64, 64, 256, 3)
    sp_corpus = zipf_csr(51 + seed, REPLICAS * n, vocab=500, mean_pairs=8)
    sp = cdb.SparseIndex(capacity_rows=REPLICAS * n, capacity_pairs=len(sp_corpus[1]))
    sp.append(sp_corpus)
    return vecs, ix, sp


def test_one_slot_group_gives_a_replica_graph_its_hybrid_search():
    vecs, ix, sp = replica_index()
    rng = np.random.default_rng(5)
    nq = 64
    q = (vecs[rng.integers(0, vecs.shape[0], nq)] + 0.02 * rng.normal(size=(nq, 32))).astype(np.float32)
    sq = zipf_csr(52, nq, vocab=500, mean_pairs=6)
    dense_opts = {"mode": cdb.SearchMode.HNSW, "ef_search": 64, "shortlist_size": 64}
    with pytest.raises(cdb.CosdataError) as e:                        # the single-handle entry point refuses it
        cdb.hybrid_batch_search(10, 60.0, dense=(ix, q, dense_opts), sparse=(sp, sq, None))
    assert e.value.status == cdb.Status.UNSUPPORTED
    g = ShardGroup.local([0])
    g.attach(0, ix)
    g.attach_sparse(0, sp)
    for top_k in (1, 10, 341):
        d_ids, _, d_counts, d_err = ix.batch_search_filtered(q, [None] * nq, 3 * top_k, ef_search=64, shortlist_size=64)
        s_ids, _, s_counts = sp.batch_search(sq, cdb.SparseSearchOptions(3 * top_k))
        got = g.hybrid_search(top_k, 60.0, dense=(q, dense_opts), sparse=(sq, None), dense_id_stride=REPLICAS)
        check(got, ph.fuse_batch(d_ids, d_counts, s_ids, s_counts, 60.0, (REPLICAS, 1), ld_out=6 * top_k))
        assert np.array_equal(got[3], d_err)
    with pytest.raises(cdb.CosdataError) as e:                        # metadata shards search in HNSW mode only
        g.hybrid_search(10, 60.0, dense=(q, {"mode": cdb.SearchMode.BRUTE_RAW}), sparse=(sq, None))
    assert e.value.status == cdb.Status.INVALID_PARAMS
    g.close(); ix.close(); sp.close()


def test_replica_group_and_mixed_group():
    from tests.test_gpu_sharded_filtered import ID_STRIDE, md_shard, plain_shard
    parts = [md_shard(s, seed=11 + s) for s in range(2)]
    shards = [p[2] for p in parts]
    sps = []
    g = ShardGroup.local([0, 0])
    for s, ix in enumerate(shards):
        g.attach(s, ix)
        corpus = zipf_csr(60 + s, 4000, vocab=400, mean_pairs=8)
        sp = cdb.SparseIndex(capacity_rows=4000, capacity_pairs=len(corpus[1]), id_base=s * ID_STRIDE)
        sp.append(corpus)
        g.attach_sparse(s, sp)
        sps.append(sp)
    vecs = parts[0][0]
    rng = np.random.default_rng(9)
    nq = 64
    q = (vecs[rng.integers(0, vecs.shape[0], nq)] + 0.02 * rng.normal(size=(nq, 24))).astype(np.float32)
    sq = zipf_csr(70, nq, vocab=400, mean_pairs=6)
    dense_opts = {"mode": cdb.SearchMode.HNSW, "ef_search": 48}
    for top_k in (1, 10, 341):
        kw, lists = group_sources(g, ("dense", "sparse"), q, sq, None, dense_opts, cdb.SparseSearchOptions(0), md=True)
        got = g.hybrid_search(top_k, 60.0, dense_id_stride=REPLICAS, **kw)
        check(got, expected(lists(top_k), top_k, (REPLICAS, 1)))
        assert np.array_equal(got[3], g.search_filtered(q, [None] * nq, 3 * top_k, ef_search=48)[3])
    g.close()
    # a replica graph next to a plain graph: one path for the dense side is not possible
    _, plain = plain_shard(1, 400, 3, 5)
    g = ShardGroup.local([0, 0])
    g.attach(0, shards[0])
    g.attach(1, plain)
    for s in range(2):
        g.attach_sparse(s, sps[s])
    with pytest.raises(cdb.CosdataError) as e:
        g.hybrid_search(10, 60.0, dense=(q, dense_opts), sparse=(sq, None))
    assert e.value.status == cdb.Status.INVALID_PARAMS and "graph metadata" in str(e.value)
    g.close()
    for x in shards + sps + [plain]:
        x.close()


# ---------------------------------------------------------------- device form
def test_device_form_equals_the_host_form():
    import torch
    w = World(1, seed=77)
    dev = torch.device("cuda", 0)
    b, top_k = 256, 10
    dq, sq, tq = w.queries(b)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view({np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(  # noqa: E731
        np.asarray(a).dtype, np.asarray(a).dtype))).to(dev)
    d_q, d_sq = t(dq), [t(a) for a in sq]
    s = torch.cuda.Stream(dev)
    for g in (ShardGroup.rank(None, 1, 0, 0), ShardGroup.local([0])):
        g.attach(0, w.raw[0])
        g.attach_sparse(0, w.sp[0])
        g.attach_tfidf(0, w.tf[0])
        for sp_opts in SPARSE_OPTS:
            host = g.hybrid_search(top_k, 60.0, dense=(dq, DENSE_TC), sparse=(sq, sp_opts))
            ids = torch.zeros((b, 6 * top_k), dtype=torch.int32, device=dev)
            sc = torch.zeros((b, 6 * top_k), dtype=torch.float32, device=dev)
            cnt = torch.zeros(b, dtype=torch.int32, device=dev)
            err = torch.full((b,), 0xEE, dtype=torch.uint8, device=dev)
            torch.cuda.synchronize(dev)
            g.hybrid_search_device(b, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), err.data_ptr(), s.cuda_stream, top_k, 60.0,
                                   dense=(d_q.data_ptr(), DENSE_TC), sparse=(tuple(x.data_ptr() for x in d_sq), sp_opts))
            s.synchronize()
            check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), host)
            assert np.array_equal(err.cpu().numpy(), host[3])
        with pytest.raises(cdb.CosdataError) as e:
            g.hybrid_search_device(b, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), None, s.cuda_stream, top_k, 60.0,
                                   sparse=(tuple(x.data_ptr() for x in d_sq), None), tfidf=(d_sq[0].data_ptr(), d_sq[1].data_ptr()))
        assert e.value.status == cdb.Status.UNSUPPORTED
        g.close()
    w.close()
