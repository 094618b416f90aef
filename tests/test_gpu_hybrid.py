"""Hybrid search on the GPU (cdb_rrf_fuse*, cdb_hybrid_search_batch*) against tests/pyhybrid.py, bit for bit (ids, counts
and score bits): the fusion kernel on random and adversarial lists (empty, one-sided, disjoint, fully overlapping, repeated
ids, id strides, ids near 2^32 - 2, up to 1023 entries per list, batch 1 and 1024) under fusion constants from 60 to NaN;
the composed search for each pairing against the fusion of the two handles' own results at k = 3 * top_k (HNSW on a
GPU-built graph, brute force on the tensor-core path, sparse with and without re-rank, deleted rows in every handle);
replica-id dense results fused with id_stride; error bytes written only with a dense source; the device form on a side stream, 8 host threads, and appends and deletes
queued behind hybrid searches.  The tests without the gpu mark check the refusals that come before any device work."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from tests import pyhybrid as ph
from tests.sparse_data import zipf_csr
from tests.tfidf_data import query_csr, zipf_docs, zipf_queries

gpu = pytest.mark.gpu
N, DIM, B, VOCAB = 20_000, 64, 64, 3000
ASSOC_K, _ = ph.association_case()


def f32_of(u):
    return np.array([u], np.uint32).view(np.float32)[0]


K_VALUES = [60.0, 0.0, 1.0, -float(ph.EPS), -3.0, -0.5, float(ASSOC_K), 1e30, 3e38, np.inf, -np.inf,
            f32_of(0xFFA00001), f32_of(0x7FC12345)]


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def check(got, want):
    ids, scores, counts = got[:3]
    w_ids, w_scores, w_counts = want
    assert np.array_equal(counts, w_counts)
    assert np.array_equal(ids, w_ids)
    assert np.array_equal(bits(scores), bits(w_scores))


# ---------------------------------------------------------------- refusals without a device (no gpu mark)
def test_fuse_refusals_come_before_the_device():
    L = _lib.load()
    ids = np.zeros(4096, np.uint32)
    cnt = np.zeros(1, np.uint32)
    out = np.zeros(4096, np.uint32)
    p = lambda a: a.ctypes.data   # noqa: E731
    assert L.cdb_rrf_fuse(0, p(ids), p(cnt), 1024, 1, p(ids), p(cnt), 1025, 1, 1, 60.0, 2049, p(out), p(out), p(cnt)) == cdb.Status.INVALID_PARAMS
    assert L.cdb_rrf_fuse(0, p(ids), p(cnt), 10, 1, p(ids), p(cnt), 10, 1, 1, 60.0, 19, p(out), p(out), p(cnt)) == cdb.Status.INVALID_PARAMS
    assert L.cdb_rrf_fuse_device(0, p(ids), p(cnt), 2000, 1, p(ids), p(cnt), 49, 1, 1, 60.0, 2049, p(out), p(out), p(cnt),
                                 None) == cdb.Status.INVALID_PARAMS
    if cdb.device_count() == 0:
        assert L.cdb_rrf_fuse(0, p(ids), p(cnt), 10, 1, p(ids), p(cnt), 10, 1, 1, 60.0, 20, p(out), p(out), p(cnt)) == cdb.Status.CUDA_ERROR
        with pytest.raises(cdb.CosdataError) as e:
            cdb.rrf_fuse(np.zeros((2, 3), np.uint32), [1, 2], np.zeros((2, 3), np.uint32), [3, 0])
        assert e.value.status == cdb.Status.CUDA_ERROR


def test_hybrid_refusals_come_before_the_handles_are_read():
    """malformed requests are refused before a handle is dereferenced: stand-in handles point at zeroed memory"""
    L = _lib.load()
    blob = (C.c_uint8 * 4096)()
    fake = C.cast(blob, C.c_void_p)
    q = np.zeros(64, np.float32)
    off = np.zeros(2, np.uint64)
    out = np.zeros(4096, np.uint32)
    cnt = np.zeros(1, np.uint32)

    def call(top_k=10, **parts):
        s = _lib.HybridSources()
        for name in parts.get("use", ()):
            setattr(s, name, fake)
            setattr(s, {"dense": "dense_queries", "sparse": "sparse_offsets", "tfidf": "tfidf_offsets"}[name],
                    q.ctypes.data if name == "dense" else off.ctypes.data)
        s.sparse_params.rerank = parts.get("rerank", 0)
        s.sparse_params.reranking_factor = parts.get("factor", 5)
        if parts.get("null_queries"):
            s.sparse_offsets = None
        return L.cdb_hybrid_search_batch(C.byref(s), 1, top_k, 60.0, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None)

    assert call(use=("sparse",)) == cdb.Status.INVALID_PARAMS                         # one source
    assert call(use=("dense", "sparse", "tfidf")) == cdb.Status.INVALID_PARAMS        # three sources
    assert call(use=()) == cdb.Status.INVALID_PARAMS
    assert call(342, use=("sparse", "tfidf")) == cdb.Status.INVALID_PARAMS            # 3 * top_k > 1024
    assert call(341, use=("sparse", "tfidf"), rerank=1, factor=6) == cdb.Status.INVALID_PARAMS   # 3 * 341 * 6 > 5120
    assert call(use=("sparse", "tfidf"), rerank=1, factor=0) == cdb.Status.INVALID_PARAMS
    assert call(use=("sparse", "tfidf"), null_queries=True) == cdb.Status.INVALID_PARAMS
    assert L.cdb_hybrid_search_batch(None, 1, 10, 60.0, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None) == cdb.Status.INVALID_PARAMS
    assert L.cdb_hybrid_search_batch_device(None, 1, 10, 60.0, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None,
                                            None) == cdb.Status.INVALID_PARAMS


# ---------------------------------------------------------------- the fusion kernel
def random_lists(rng, nq, ld, id_range, dup=0.2, top=None):
    ids = rng.integers(0, id_range, (nq, ld)).astype(np.uint64)
    if top is not None:
        ids = np.uint64(top) - ids
    ids = ids.astype(np.uint32)
    counts = rng.integers(0, ld + 1, nq).astype(np.uint32)
    counts[rng.random(nq) < 0.3] = ld
    return ids, counts


def fuse_both(a, ca, b, cb, k, strides=(1, 1)):
    got = cdb.rrf_fuse(a, ca, b, cb, k, strides)
    want = ph.fuse_batch(a, ca, b, cb, k, strides)
    check(got, want)
    return got


@gpu
@pytest.mark.parametrize("k", K_VALUES, ids=lambda k: f"{np.float32(k).view(np.uint32):08x}")
def test_fusion_kernel_random_and_adversarial_lists(k):
    rng = np.random.default_rng(int(np.float32(k).view(np.uint32)) & 0xFFFF)
    # B = 1024, short lists with many repeated ids, each stride
    for stride in (1, 4, 16):
        a, ca = random_lists(rng, 1024, 30, 60)
        b, cb = random_lists(rng, 1024, 30, 60)
        fuse_both(a, ca, b, cb, k, (stride, stride))
    # long lists at B = 1 and B = 4, ids near 2^32 - 2 (and 2^32 - 1 taken as given)
    a, ca = random_lists(rng, 4, 1023, 3000, top=0xFFFFFFFF)
    b, cb = random_lists(rng, 4, 1023, 3000, top=0xFFFFFFFF)
    fuse_both(a, ca, b, cb, k, (1, 16))
    fuse_both(a[:1], ca[:1], b[:1], cb[:1], k)
    r = np.arange(500, dtype=np.uint32)
    one = np.ones(1, np.uint32)
    full = lambda x: np.array([len(x)], np.uint32)   # noqa: E731
    cases = [
        (r[None, :0], one * 0, r[None, :0], one * 0),                     # both empty (ld 0)
        (r[None, :10], one * 0, r[None, :7], one * 0),                     # counts 0
        (r[None, :300], full(r[:300]), r[None, :0], one * 0),              # one-sided
        (r[None, :0], one * 0, r[None, :300], full(r[:300])),
        (r[None, :250], full(r[:250]), r[None, 250:], full(r[250:])),      # disjoint
        (r[None, :400], full(r[:400]), r[None, ::-1][:, 100:], full(r[100:])),   # full overlap, reversed ranks
        (np.full((1, 20), 7, np.uint32), one * 20, np.full((1, 20), 7, np.uint32), one * 20),   # one id everywhere
        (np.array([[0xFFFFFFFE, 0xFFFFFFFD, 0xFFFFFFFE, 0]], np.uint32), one * 4,
         np.array([[0, 0xFFFFFFFF, 0xFFFFFFFE]], np.uint32), one * 3),
    ]
    for a, ca, b, cb in cases:
        for strides in ((1, 1), (4, 16)):
            fuse_both(a, ca, b, cb, k, strides)


@gpu
def test_fusion_kernel_device_form_on_a_side_stream():
    import torch
    rng = np.random.default_rng(8)
    a, ca = random_lists(rng, 1024, 200, 400)
    b, cb = random_lists(rng, 1024, 90, 400)
    want = ph.fuse_batch(a, ca, b, cb, 60.0, (1, 4))
    dev = torch.device("cuda", 0)
    t = lambda x: torch.from_numpy(x.astype(np.int32)).to(dev)   # noqa: E731
    da, dca, db, dcb = t(a), t(ca), t(b), t(cb)
    ids = torch.zeros((1024, 290), dtype=torch.int32, device=dev)
    sc = torch.zeros((1024, 290), dtype=torch.float32, device=dev)
    cnt = torch.zeros(1024, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    assert _lib.load().cdb_rrf_fuse_device(0, da.data_ptr(), dca.data_ptr(), 200, 1, db.data_ptr(), dcb.data_ptr(), 90, 4, 1024, 60.0,
                                           290, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), C.c_void_p(s.cuda_stream)) == 0
    s.synchronize()
    check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), want)


# ---------------------------------------------------------------- the composed search
@pytest.fixture(scope="module")
def world():
    """one id space, N rows in every handle: a dense HNSW handle (graph built on the GPU), a dense f32 handle for the
    brute-force tensor-core path, a sparse and a TF-IDF handle; every handle has deleted rows"""
    rng = np.random.default_rng(31)
    centres = rng.normal(size=(64, DIM)).astype(np.float32)
    vecs = (centres[rng.integers(0, 64, N)] + 0.4 * rng.normal(size=(N, DIM))).astype(np.float32)
    vecs /= np.abs(vecs).max() * 1.01
    hn = cdb.DenseIndex(dim=DIM, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=N + 1, keep_raw_f32=True)
    hn.append(vecs)
    hn.build_graph(num_levels=4, neighbors_count=16, level0_neighbors_count=32, ef_construction=64, shortlist_size=32)
    hn.delete_rows(rng.choice(N, 300, replace=False))
    raw = cdb.DenseIndex(dim=DIM, capacity=N, tensor_prefilter=True)
    raw.append(vecs)
    raw.delete_rows(rng.choice(N, 300, replace=False))
    sp_corpus = zipf_csr(41, N, vocab=VOCAB, mean_pairs=24)
    sp = cdb.SparseIndex(capacity_rows=N, capacity_pairs=len(sp_corpus[1]))
    sp.append(sp_corpus)
    sp.delete_embedding(rng.choice(N, 300, replace=False))
    tf_corpus = zipf_docs(42, N, vocab=VOCAB, mean_terms=16)
    tf = cdb.TfIdfIndex(capacity_rows=N, capacity_pairs=len(tf_corpus[1]))
    tf.append(tf_corpus, 1)
    tf.delete_embedding(rng.choice(N, 300, replace=False), 2)
    dq = (vecs[rng.integers(0, N, B)] + 0.05 * rng.normal(size=(B, DIM))).astype(np.float32)
    sq = zipf_csr(43, B, vocab=VOCAB, mean_pairs=10)
    tq = zipf_queries(44, B, vocab=VOCAB)
    w = dict(hn=hn, raw=raw, sp=sp, tf=tf, dq=dq, sq=sq, tq=tq)
    yield w
    for h in (hn, raw, sp, tf):
        h.close()


DENSE_HNSW = {"mode": cdb.SearchMode.HNSW, "ef_search": 256, "shortlist_size": 64}
DENSE_TC = {"mode": cdb.SearchMode.BRUTE_RAW, "tensor_with_deleted": True}


def sources(w, pair, rerank=False, dense_handle="hn", dense_opts=DENSE_HNSW):
    """-> (kwargs of hybrid_batch_search, function top_k -> the two lists (ids, scores, counts) the handles return)"""
    kw, run = {}, {}
    sp_opts = lambda k3: cdb.SparseSearchOptions(k3, None, rerank, 5)   # noqa: E731
    if "dense" in pair:
        ix = w[dense_handle]
        kw["dense"] = (ix, w["dq"], dense_opts)
        run["dense"] = lambda k3: ix.batch_search(w["dq"], k3, **dense_opts)[:3]
    if "sparse" in pair:
        kw["sparse"] = (w["sp"], w["sq"], sp_opts(0))
        run["sparse"] = lambda k3: w["sp"].batch_search(w["sq"], sp_opts(k3))
    if "tfidf" in pair:
        kw["tfidf"] = (w["tf"], w["tq"])
        run["tfidf"] = lambda k3: w["tf"].batch_search(w["tq"], k3)
    return kw, lambda top_k: (run[pair[0]](3 * top_k), run[pair[1]](3 * top_k))


def expected(lists, top_k, k=60.0):
    (a, _, ca), (b, _, cb) = lists
    return ph.fuse_batch(a, ca, b, cb, k, ld_out=6 * top_k)


PAIRS = [("dense", "sparse"), ("dense", "tfidf"), ("sparse", "tfidf")]


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids="-".join)
@pytest.mark.parametrize("top_k", [1, 10, 200, 341])
@pytest.mark.parametrize("rerank", [False, True], ids=["plain", "rerank"])
def test_composed_search_equals_the_fusion_of_its_sources(world, pair, top_k, rerank):
    if rerank and "sparse" not in pair:
        pytest.skip("re-rank is a sparse option")
    kw, lists = sources(world, pair, rerank)
    got = cdb.hybrid_batch_search(top_k, 60.0, **kw)
    src = lists(top_k)
    check(got, expected(src, top_k))
    assert got[0].shape == (B, 6 * top_k)
    assert (got[2] > top_k).any()                            # the union, not truncated to top_k
    if "dense" in pair:
        assert np.array_equal(got[3], world["hn"].batch_search(world["dq"], 3 * top_k, **DENSE_HNSW)[3])
    else:
        assert not got[3].any()
    # every handle has deleted rows, and none of them came back from its own search
    handle = {"dense": (world["hn"], lambda h: np.flatnonzero(h.deleted_rows())),
              "sparse": (world["sp"], lambda h: np.flatnonzero(h.deleted_rows()[0])),
              "tfidf": (world["tf"], lambda h: np.flatnonzero(h.deleted_rows()[0]))}
    for name, (ids, _, counts) in zip(pair, src):
        h, dead = handle[name]
        dead = set(dead(h).tolist())
        assert len(dead) == 300
        assert not dead & {int(i) for row, c in zip(ids, counts) for i in row[:c]}


@gpu
@pytest.mark.parametrize("pair", PAIRS[:2], ids="-".join)
@pytest.mark.parametrize("top_k", [1, 10, 21])
def test_composed_search_with_brute_force_on_the_tensor_core_path(world, pair, top_k):
    kw, lists = sources(world, pair, dense_handle="raw", dense_opts=DENSE_TC)
    before = world["raw"].stats()["tensor_searches"]
    got = cdb.hybrid_batch_search(top_k, 60.0, **kw)
    assert world["raw"].stats()["tensor_searches"] == before + 1
    check(got, expected(lists(top_k), top_k))


@gpu
@pytest.mark.parametrize("k", [0.0, -3.0, float(ASSOC_K), 3e38, -np.inf, f32_of(0xFFA00001)],
                         ids=lambda k: f"{np.float32(k).view(np.uint32):08x}")
def test_composed_search_under_edge_fusion_constants(world, k):
    kw, lists = sources(world, ("sparse", "tfidf"))
    check(cdb.hybrid_batch_search(10, k, **kw), expected(lists(10), 10, k))


@gpu
def test_top_k_limits(world):
    kw, _ = sources(world, ("dense", "sparse"))
    with pytest.raises(cdb.CosdataError) as e:
        cdb.hybrid_batch_search(342, 60.0, **kw)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    n0 = cdb.kernel_launch_count()
    ids, scores, counts, err = cdb.hybrid_batch_search(0, 60.0, **kw)
    assert cdb.kernel_launch_count() == n0
    assert ids.shape == (B, 0) and not counts.any()
    with pytest.raises(cdb.CosdataError) as e:                # the sparse search's own limit, refused up front
        cdb.hybrid_batch_search(341, 60.0, sparse=(world["sp"], world["sq"], cdb.SparseSearchOptions(0, None, True, 6)),
                                tfidf=(world["tf"], world["tq"]))
    assert e.value.status == cdb.Status.INVALID_PARAMS


@gpu
def test_replica_id_dense_results_fuse_with_id_stride():
    from tests import mdgraph
    replicas = 4                                              # mdgraph.replica_population's ids: i * 4 + j
    pop = mdgraph.replica_population(n=2000, dim=32, md_dims=6, levels=4, seed=7)
    vecs = pop["vecs"]
    n = vecs.shape[0]
    ix = cdb.DenseIndex(dim=32, storage_type=cdb.StorageType.HalfPrecisionFP, capacity=n + 2, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph_replicas(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], pop["md_bits"],
                            pop["md_mags"], pop["main_root_md"], pop["pseudo_root_md"], 4, 16, 32, 64, 64, 256, 3)
    rng = np.random.default_rng(5)
    nq, top_k = 16, 10
    q = (vecs[rng.integers(0, n, nq)] + 0.02 * rng.normal(size=(nq, 32))).astype(np.float32)
    d_ids, _, d_counts, _ = ix.batch_search_filtered(q, [None] * nq, 3 * top_k, ef_search=64, shortlist_size=64)
    # unfiltered searches start at the main root and return base replicas (i * replicas)
    assert all(int(i) % replicas == 0 for row, c in zip(d_ids, d_counts) for i in row[:c])
    sp_corpus = zipf_csr(51, replicas * n, vocab=500, mean_pairs=8)
    sp = cdb.SparseIndex(capacity_rows=replicas * n, capacity_pairs=len(sp_corpus[1]))
    sp.append(sp_corpus)
    sq = zipf_csr(52, nq, vocab=500, mean_pairs=6)
    s_ids, _, s_counts = sp.batch_search(sq, cdb.SparseSearchOptions(3 * top_k))
    check(cdb.rrf_fuse(d_ids, d_counts, s_ids, s_counts, 60.0, (replicas, 1)),
          ph.fuse_batch(d_ids, d_counts, s_ids, s_counts, 60.0, (replicas, 1)))
    # filtered searches reach the metadata replicas (i * replicas + j): the stride folds them onto their embedding's key
    filters = [[pop["md_bits"][2 + i % 7].astype(np.int8)] for i in range(nq)]
    f_ids, _, f_counts, _ = ix.batch_search_filtered(q, filters, 3 * top_k, ef_search=64, shortlist_size=64)
    assert any(int(i) % replicas for row, c in zip(f_ids, f_counts) for i in row[:c])
    got = cdb.rrf_fuse(f_ids, f_counts, s_ids, s_counts, 60.0, (replicas, 1))
    check(got, ph.fuse_batch(f_ids, f_counts, s_ids, s_counts, 60.0, (replicas, 1)))
    with pytest.raises(cdb.CosdataError) as e:
        cdb.hybrid_batch_search(top_k, 60.0, dense=(ix, q, DENSE_HNSW), sparse=(sp, sq, None))
    assert e.value.status == cdb.Status.UNSUPPORTED
    ix.close()
    sp.close()


# ---------------------------------------------------------------- concurrency
def device_sources(w, pair, dev):
    """cdb_hybrid_sources over device copies of the queries -> (struct, tensors to keep alive)"""
    import torch
    src, keep = _lib.HybridSources(), []

    def put(a):
        a = np.ascontiguousarray(a)
        t = torch.from_numpy(a.view({np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(a.dtype, a.dtype))).to(dev)
        keep.append(t)
        return t.data_ptr()
    if "dense" in pair:
        src.dense, src.dense_queries, src.dense_params = w["hn"]._h, put(w["dq"]), w["hn"].params(0, **DENSE_HNSW)
    if "sparse" in pair:
        o, d, v = w["sq"]
        src.sparse, src.sparse_offsets, src.sparse_dims, src.sparse_values = w["sp"].h, put(o), put(d), put(v)
        src.sparse_params = cdb.SparseSearchOptions(0).params()
    if "tfidf" in pair:
        o, h = query_csr(w["tq"])
        src.tfidf, src.tfidf_offsets, src.tfidf_hashes = w["tf"].h, put(o), put(h)
    return src, keep


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids="-".join)
def test_device_form_on_a_side_stream_and_threads(world, pair):
    import torch
    dev = torch.device("cuda", 0)
    kw, lists = sources(world, pair)
    want = expected(lists(10), 10)
    src, alive = device_sources(world, pair, dev)
    s = torch.cuda.Stream(dev)
    ids = torch.zeros((B, 60), dtype=torch.int32, device=dev)
    sc = torch.zeros((B, 60), dtype=torch.float32, device=dev)
    cnt = torch.zeros(B, dtype=torch.int32, device=dev)
    err = torch.zeros(B, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    assert _lib.load().cdb_hybrid_search_batch_device(C.byref(src), B, 10, 60.0, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                                                      err.data_ptr(), C.c_void_p(s.cuda_stream)) == 0
    s.synchronize()
    check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), want)
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        for got in ex.map(lambda _: cdb.hybrid_batch_search(10, 60.0, **kw), range(16)):
            check(got, want)


@gpu
@pytest.mark.parametrize("pair", PAIRS, ids="-".join)
def test_error_bytes_only_with_a_dense_source(world, pair):
    """0xEE-filled err_flags get the dense search's bytes with a dense source and stay untouched without one, in the host
    and the device form"""
    import torch
    from cosdata_b200.api import hybrid_sources
    dev = torch.device("cuda", 0)
    kw, _ = sources(world, pair)
    want = world["hn"].batch_search(world["dq"], 30, **DENSE_HNSW)[3] if "dense" in pair else np.full(B, 0xEE, np.uint8)
    src, keep, _ = hybrid_sources(**kw)
    ids, sc = np.zeros((B, 60), np.uint32), np.zeros((B, 60), np.float32)
    cnt, err = np.zeros(B, np.uint32), np.full(B, 0xEE, np.uint8)
    assert _lib.load().cdb_hybrid_search_batch(C.byref(src), B, 10, 60.0, ids.ctypes.data, sc.ctypes.data, cnt.ctypes.data,
                                               err.ctypes.data) == 0
    assert np.array_equal(err, want)
    src, alive = device_sources(world, pair, dev)
    ids = torch.zeros((B, 60), dtype=torch.int32, device=dev)
    sc = torch.zeros((B, 60), dtype=torch.float32, device=dev)
    cnt = torch.zeros(B, dtype=torch.int32, device=dev)
    err = torch.full((B,), 0xEE, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    assert _lib.load().cdb_hybrid_search_batch_device(C.byref(src), B, 10, 60.0, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                                                      err.data_ptr(), None) == 0
    torch.cuda.synchronize(dev)
    assert np.array_equal(err.cpu().numpy(), want)


@gpu
def test_append_and_delete_queued_behind_hybrid_searches():
    """searches enqueued on a stream before an append and a delete see the handles as they were"""
    import torch
    dev = torch.device("cuda", 0)
    n0, n1 = 12_000, 16_000
    sp_corpus = zipf_csr(61, n1, vocab=VOCAB, mean_pairs=24)
    tf_corpus = zipf_docs(62, n1, vocab=VOCAB, mean_terms=16)
    head = lambda c: (c[0][:n0 + 1], *(x[:int(c[0][n0])] for x in c[1:]))   # noqa: E731
    tail = lambda c: (c[0][n0:] - c[0][n0], *(x[int(c[0][n0]):] for x in c[1:]))   # noqa: E731
    sp = cdb.SparseIndex(capacity_rows=n1, capacity_pairs=len(sp_corpus[1]))
    tf = cdb.TfIdfIndex(capacity_rows=n1, capacity_pairs=len(tf_corpus[1]))
    sp.append(head(sp_corpus))
    tf.append(head(tf_corpus), 1)
    w = dict(sp=sp, tf=tf, sq=zipf_csr(63, B, vocab=VOCAB, mean_pairs=10), tq=zipf_queries(64, B, vocab=VOCAB))
    kw, lists = sources(w, ("sparse", "tfidf"))
    want = expected(lists(10), 10)
    src, alive = device_sources(w, ("sparse", "tfidf"), dev)
    s = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    outs = []
    for _ in range(8):
        ids = torch.zeros((B, 60), dtype=torch.int32, device=dev)
        sc = torch.zeros((B, 60), dtype=torch.float32, device=dev)
        cnt = torch.zeros(B, dtype=torch.int32, device=dev)
        assert _lib.load().cdb_hybrid_search_batch_device(C.byref(src), B, 10, 60.0, ids.data_ptr(), sc.data_ptr(),
                                                          cnt.data_ptr(), None, C.c_void_p(s.cuda_stream)) == 0
        outs.append((ids, sc, cnt))
    sp.append(tail(sp_corpus))
    tf.delete_embedding(np.arange(0, n0, 3, dtype=np.uint32), 2)
    s.synchronize()
    for ids, sc, cnt in outs:
        check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), want)
    after = cdb.hybrid_batch_search(10, 60.0, **kw)
    check(after, expected(lists(10), 10))
    assert not np.array_equal(after[0], want[0])
    sp.close()
    tf.close()
