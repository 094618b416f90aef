"""cdb_index_insert_graph: rows appended after a build / upload go into the live graph on the GPU.
  * one row at a time it equals the insert oracle (tests/hnsw_insert_oracle.c) array for array, slot scores included,
    after a GPU build (kept state) and after an upload (state derived by hnsw_slot_state_kernel, reload semantics);
  * the derived slot similarities equal the builder's retained ones bit for bit;
  * batched inserts keep the graph's invariants, CUDA search equals the oracle's on the grown graph, recall holds."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from tests import pyinsert

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
EMPTY = 0xFFFFFFFF


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def clustered(n, dim, seed):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(32, dim)).astype(np.float32)
    v = (centres[rng.integers(0, 32, n)] + 0.35 * rng.normal(size=(n, dim))).astype(np.float32)
    return (v / (np.abs(v).max() * 1.01)).astype(np.float32)


def assert_graph_equal(g, e, scores=None, metric=None):
    assert g["entry"] == e["entry"] and g["root_row"] == e["root_row"]
    for lv in range(g["num_levels"] + 1):
        assert np.array_equal(g["node_row"][lv], e["node_row"][lv]), lv
        assert np.array_equal(g["adj"][lv], e["adj"][lv]), lv
        if lv:
            assert np.array_equal(g["child"][lv], e["child"][lv]), lv
        if scores is not None:
            assert np.array_equal(bits(scores[lv]), bits(pyinsert.slot_scores(metric, e["simkey"][lv], e["adj"][lv]))), lv


def grown_index(vecs, n0, st, metric, levels, nb, nb0, efc, seed, max_batch=1, chunks=(), max_level=None, extra=0):
    n, dim = vecs.shape
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1 + extra, keep_raw_f32=True)
    ix.append(vecs[:n0])
    ix.build_graph(levels, nb, nb0, efc, 64, max_batch, seed)
    first = n0
    for c in chunks:
        ix.append(vecs[first:first + c])
        lv = None if max_level is None else max_level[first - n0:first - n0 + c]
        failed = ix.insert_graph(efc, 64, max_batch, seed, max_level=lv)
        assert failed.size == c and failed.sum() == 0
        first += c
    return ix


@pytest.mark.parametrize("st,metric,draws", [(ST.HalfPrecisionFP, MK.Cosine, False), (ST.UnsignedByte, MK.Cosine, False),
                                              (ST.SubByte2, MK.DotProduct, False), (ST.HalfPrecisionFP, MK.Cosine, True)])
def test_sequential_insert_equals_oracle_after_build_and_after_upload(st, metric, draws):
    n0, dim, levels, nb, nb0, efc, seed = 900, 32, 4, 8, 16, 32, 5
    vecs = clustered(n0 + 300, dim, 11)
    max_level = np.random.default_rng(3).integers(0, 3, 300).astype(np.uint8) if draws else None
    ix = grown_index(vecs, n0, st, metric, levels, nb, nb0, efc, seed, chunks=(200, 100), max_level=max_level)
    g, sc = ix.read_graph(), ix.read_graph_slot_scores()
    assert g["root_row"] == n0 and len(ix) == n0 + 301
    codes, mags = ix.read_codes(0, n0 + 301)
    o = pyinsert.Graph.init(int(metric), int(st), dim, codes, mags, n0, levels, nb, nb0)
    o.insert(0, n0, ef_construction=efc, seed=seed)
    o.insert(n0 + 1, 200, ef_construction=efc, seed=seed, max_level=None if max_level is None else max_level[:200])
    o.insert(n0 + 201, 100, ef_construction=efc, seed=seed, max_level=None if max_level is None else max_level[200:])
    assert_graph_equal(g, o.export(), sc, int(metric))
    # the same rows inserted into the uploaded first build: reload semantics (lowest_index recomputed, not stale)
    up = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 301, keep_raw_f32=True)
    base = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 1, keep_raw_f32=True)
    base.append(vecs[:n0])
    base.build_graph(levels, nb, nb0, efc, 64, 1, seed)
    g0 = base.read_graph()
    up.append(np.concatenate([vecs[:n0], root_vector(seed, dim)[None], vecs[n0:]]))
    up.set_graph(g0["num_levels"], nb, nb0, g0["entry"], g0["root_row"], g0["node_row"], g0["adj"], g0["child"])
    failed = up.insert_graph(efc, 64, 1, seed, max_level=max_level)
    assert failed.size == 300 and failed.sum() == 0
    gu, scu = up.read_graph(), up.read_graph_slot_scores()
    ucodes, umags = up.read_codes(0, n0 + 301)
    assert np.array_equal(ucodes, codes) and np.array_equal(bits(umags), bits(mags))
    ou = pyinsert.Graph.from_graph(int(metric), int(st), dim, codes, mags, g0)
    ou.insert(n0 + 1, 300, ef_construction=efc, seed=seed, max_level=max_level)
    assert_graph_equal(gu, ou.export(), scu, int(metric))
    # both paths were exercised: the stale and the recomputed lowest_index lead to different graphs
    assert any(not np.array_equal(g["adj"][lv], gu["adj"][lv]) for lv in range(levels + 1))
    for x in (ix, up, base):
        x.close()
    o.close()
    ou.close()


def root_vector(seed, dim, lo=-1.0, hi=1.0):   # the root the build appends (vector_store.rs:57-64)
    s = orc.synth(seed ^ 0x526F6F74, 0, dim)
    return (np.float32(lo) + (s + np.float32(1.0)) * np.float32(0.5) * np.float32(hi - lo)).astype(np.float32)


@pytest.mark.parametrize("n,dim,st", [(6000, 48, ST.HalfPrecisionFP), (6000, 64, ST.UnsignedByte), (50000, 768, ST.HalfPrecisionFP)])
def test_slot_state_kernel_matches_retained_state(n, dim, st):
    vecs = clustered(n, dim, 21)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=MK.Cosine, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(5, 16, 32, 64, 64, 256, 9)
    g, kept = ix.read_graph(), ix.read_graph_slot_scores()
    codes, mags = ix.read_codes(0, n + 1)
    up = cdb.DenseIndex(dim=dim, storage_type=st, metric=MK.Cosine, capacity=n + 1)
    up.append_codes(codes, mags)
    up.set_graph(g["num_levels"], 16, 32, g["entry"], g["root_row"], g["node_row"], g["adj"], g["child"])
    derived = up.read_graph_slot_scores()
    filled_total = 0
    for lv in range(6):
        filled = g["adj"][lv] != EMPTY
        filled_total += int(filled.sum())
        assert np.array_equal(bits(derived[lv])[filled], bits(kept[lv])[filled]), lv
        assert (bits(derived[lv])[~filled] == 0).all()
    assert filled_total > n * 10
    # the oracle's reload derives the same similarities
    o = pyinsert.Graph.from_graph(0, int(st), dim, codes, mags, g)
    e = o.export()
    for lv in range(6):
        assert np.array_equal(bits(derived[lv]), bits(pyinsert.slot_scores(0, e["simkey"][lv], e["adj"][lv]))), lv
    o.close()
    ix.close()
    up.close()


def test_zero_norm_rows_edges_and_errors():
    n0, dim = 500, 16
    vecs = clustered(n0 + 40, dim, 4)
    vecs[n0 + 3] = 0.0
    vecs[n0 + 17] = 0.0
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.HalfPrecisionFP, metric=MK.Cosine, capacity=n0 + 41, keep_raw_f32=True)
    ix.append(vecs[:n0])
    ix.build_graph(3, 8, 16, 32, 64, 64, 2)
    assert ix.insert_graph(32, 64, 64, 2).size == 0                      # no new rows: CDB_OK, nothing inserted
    ix.append(vecs[n0:])
    bp = cdb._lib.BuildParams(4, 8, 16, 32, 64, 64, 2)                  # num_levels differs from the graph's
    import ctypes as C
    rc = ix._lib.cdb_index_insert_graph(ix._h, C.byref(bp), None, None, None)
    assert rc == int(cdb.Status.INVALID_PARAMS)
    failed = ix.insert_graph(32, 64, 64, 2)
    assert np.flatnonzero(failed).tolist() == [3, 17]
    g = ix.read_graph()
    for bad in (n0 + 1 + 3, n0 + 1 + 17):
        assert (g["adj"][0].reshape(-1, 16)[bad] == EMPTY).all()
        assert not (g["adj"][0] == bad).any()
    ix.close()


def test_uploaded_edge_to_a_zero_norm_row_is_evicted_first():
    dim = 8
    vecs = clustered(6, dim, 1)
    vecs[2] = 0.0
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.HalfPrecisionFP, metric=MK.Cosine, capacity=9, keep_raw_f32=True)
    ix.append(np.concatenate([vecs, vecs[:1] * 0.5]))                  # row 6: the root
    nb0 = 4
    adj = np.full((7, nb0), EMPTY, np.uint32)
    # node 0 is full; its last slot links the zero-norm row 2 (a pair the reference cannot score), which a traversal with
    # shortlist 3 never reaches
    adj[0] = [1, 3, 4, 2]
    adj[1, 0], adj[3, 0], adj[4, 0], adj[6, 0], adj[6, 1] = 0, 0, 0, 0, 1
    ix.set_graph(0, 4, nb0, 6, 6, [np.arange(7, dtype=np.uint32)], [adj.ravel()], [np.zeros(7, np.uint32)])
    sc = ix.read_graph_slot_scores()[0].reshape(7, nb0)
    assert bits(sc[0, 3]) == bits(np.float32(-1.0)) and (sc[0, :3] > -1.0).all() and sc[1, 1] == 0
    ix.append(vecs[:1] * 0.9 + 0.01)                                     # close to row 0
    assert ix.insert_graph(16, 3, 1, 1).tolist() == [0]
    a0 = ix.read_graph()["adj"][0].reshape(8, nb0)[0]
    assert a0.tolist() == [1, 3, 4, 7]                                   # the Err slot was the one replaced


def test_graph_with_metadata_is_unsupported():
    from tests import mdgraph
    pop = mdgraph.replica_population(n=200, dim=16, md_dims=4, levels=2, seed=3)
    n, dim = pop["vecs"].shape
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.HalfPrecisionFP, metric=MK.Cosine, capacity=n + 3, keep_raw_f32=True)
    ix.append(pop["vecs"])
    ix.build_graph_replicas(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], pop["md_bits"],
                            pop["md_mags"], pop["main_root_md"], pop["pseudo_root_md"], 2, 8, 16, 16, 64, 64, 1)
    ix.append(pop["vecs"][:1])
    with pytest.raises(cdb.CosdataError) as e:
        ix.insert_graph(16, 64, 64, 1)
    assert e.value.status == cdb.Status.UNSUPPORTED
    ix.close()


def test_batched_insert_invariants_search_parity_and_recall():
    n0, dim, k = 5000, 48, 10
    vecs = clustered(n0 + 2000, dim, 21)
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    rng = np.random.default_rng(2)
    queries = (vecs[rng.integers(0, n0 + 2000, 64)] + 0.05 * rng.normal(size=(64, dim))).astype(np.float32)
    one = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 2001, keep_raw_f32=True)
    one.append(vecs)
    one.build_graph(5, 16, 32, 64, 64, 256, 9)
    ids1, _, _, _ = one.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=64, shortlist_size=64)
    recalls = {}
    for name, chunks in (("one", (1000, 1000)), ("ten", (1000,) + (100,) * 10)):
        ix = grown_index(vecs, n0, st, metric, 5, 16, 32, 64, 9, max_batch=256, chunks=chunks)
        g = ix.read_graph()
        n = n0 + 2001
        assert g["root_row"] == n0 and np.array_equal(g["node_row"][0], np.arange(n, dtype=np.uint32))
        for lv in range(6):
            nbc = 32 if lv == 0 else 16
            adj = g["adj"][lv].reshape(-1, nbc)
            valid = adj[adj != EMPTY]
            assert valid.size == 0 or valid.max() < adj.shape[0]
            assert not np.any(adj == np.arange(adj.shape[0], dtype=np.uint32)[:, None])
            for i in range(0, adj.shape[0], 7):
                row = adj[i][adj[i] != EMPTY]
                assert row.size == np.unique(row).size
            if lv >= 1:
                assert g["node_row"][lv][0] == n0
                assert np.array_equal(g["node_row"][lv - 1][g["child"][lv]], g["node_row"][lv])
        deg0 = (g["adj"][0].reshape(-1, 32) != EMPTY).sum(1)
        assert (deg0[n0 + 1:] > 0).mean() > 0.99
        codes, mags = ix.read_codes(0, n)
        raw = np.concatenate([vecs[:n0], np.zeros((1, dim), np.float32), vecs[n0:]])
        ev0, _ = ix.hnsw_counters()
        ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=64, shortlist_size=64)
        ev1, _ = ix.hnsw_counters()
        o = pyinsert.Graph.from_graph(int(metric), int(st), dim, codes, mags, g)
        w = o.search_batch(raw, queries, k, ef_search=64)
        o.close()
        gids = np.where(ids > n0, ids - 1, ids)   # rows -> positions in vecs (the root sits at row n0)
        assert np.array_equal(ids, w[0]) and np.array_equal(bits(scores), bits(w[1])) and np.array_equal(counts, w[2])
        assert ev1 - ev0 == w[4]
        gt, _ = orc.brute_topk_f32(vecs, queries, k)
        recalls[name] = np.mean([len(set(gids[i]) & set(gt[i])) / k for i in range(len(queries))])
        ix.close()
    gt, _ = orc.brute_topk_f32(vecs, queries, k)
    r1 = np.mean([len(set(ids1[i]) & set(gt[i])) / k for i in range(len(queries))])
    for name, r in recalls.items():
        assert r >= 0.85 and r >= r1 - 0.05, (name, r, r1)
    one.close()


def test_searches_before_and_after_an_insert_see_the_old_and_the_new_graph():
    # a search thread enqueues a device search on its own stream, the main thread inserts, then the search thread enqueues
    # another search on a second stream: the first must return the old graph's results, the second the new graph's
    import threading
    import torch
    n0, n1, dim, k, nq = 4000, 1000, 48, 10, 512
    vecs = clustered(n0 + n1, dim, 31)
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + n1 + 1, keep_raw_f32=True)
    ix.append(vecs[:n0])
    ix.build_graph(5, 16, 32, 64, 64, 256, 9)
    ix.append(vecs[n0:])
    old = ix.read_graph()
    rng = np.random.default_rng(6)
    queries = (vecs[rng.integers(0, n0 + n1, nq)] + 0.05 * rng.normal(size=(nq, dim))).astype(np.float32)
    dq = torch.from_numpy(queries).cuda()
    out = [(torch.empty((nq, k), dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
            torch.empty(nq, dtype=torch.int32, device="cuda")) for _ in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    enqueued, inserted, errors = threading.Event(), threading.Event(), []

    def searcher():
        try:
            for i in range(2):
                if i == 1:
                    inserted.wait()
                ids, sc, cnt = out[i]
                ix.batch_search_device(dq.data_ptr(), nq, k, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                                       stream_ptr=streams[i].cuda_stream, mode=cdb.SearchMode.HNSW, ef_search=64, shortlist_size=64)
                enqueued.set()
        except Exception as e:   # surfaced by the main thread
            errors.append(e)
            enqueued.set()

    t = threading.Thread(target=searcher)
    t.start()
    enqueued.wait()
    failed = ix.insert_graph(64, 64, 256, 9)
    inserted.set()
    t.join()
    assert not errors and failed.size == n1 and failed.sum() == 0
    for s_ in streams:
        s_.synchronize()
    new = ix.read_graph()
    codes, mags = ix.read_codes(0, n0 + n1 + 1)
    raw = np.concatenate([vecs[:n0], np.zeros((1, dim), np.float32), vecs[n0:]])
    for graph, (ids, sc, cnt) in zip((old, new), out):
        o = pyinsert.Graph.from_graph(int(metric), int(st), dim, codes, mags, graph)
        w = o.search_batch(raw, queries, k, ef_search=64)
        o.close()
        assert np.array_equal(ids.cpu().numpy().view(np.uint32), w[0])
        assert np.array_equal(bits(sc.cpu().numpy()), bits(w[1])) and np.array_equal(cnt.cpu().numpy().view(np.uint32), w[2])
    # the two graphs answer differently: the new rows are reachable only in the second
    assert not np.array_equal(out[0][0].cpu().numpy(), out[1][0].cpu().numpy())
    assert (out[1][0].cpu().numpy().view(np.uint32) > n0).any() and not (out[0][0].cpu().numpy().view(np.uint32) > n0).any()
    ix.close()
