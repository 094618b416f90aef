"""cdb_index_delete_rows: delete_embedding on the GPU (graph repair with the deviations D1-D4) and deleted rows skipped by
the exact scans.
  * one row at a time it equals the delete oracle (tests/hnsw_delete_oracle.c) array for array, slot scores and statuses
    included, after a GPU build and after an upload, and through an interleaved build / delete / append / insert flow;
  * batched deletes leave no link to a deleted row, keep every slot's similarity exact, and CUDA search on the repaired
    graph equals the oracle's; recall stays close to a fresh build over the live rows;
  * no search mode returns a deleted row; brute-force modes equal the oracle's scan over the live rows;
  * refusals change nothing; build and insert skip deleted rows; searches enqueued before a delete see the old graph."""
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from tests import pydelete, pyinsert

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


def root_vector(seed, dim, lo=-1.0, hi=1.0):   # the root the build appends (vector_store.rs:57-64)
    s = orc.synth(seed ^ 0x526F6F74, 0, dim)
    return (np.float32(lo) + (s + np.float32(1.0)) * np.float32(0.5) * np.float32(hi - lo)).astype(np.float32)


def assert_graph_equal(g, e, scores, metric):
    assert g["entry"] == e["entry"] and g["root_row"] == e["root_row"]
    for lv in range(g["num_levels"] + 1):
        assert np.array_equal(g["node_row"][lv], e["node_row"][lv]), lv
        assert np.array_equal(g["adj"][lv], e["adj"][lv]), lv
        if lv:
            assert np.array_equal(g["child"][lv], e["child"][lv]), lv
        assert np.array_equal(bits(scores[lv]), bits(pyinsert.slot_scores(metric, e["simkey"][lv], e["adj"][lv]))), lv


def assert_unlinked(g, deleted_rows):
    dead = np.zeros(int(max(g["node_row"][0].max(), max(deleted_rows, default=0))) + 1, bool)
    dead[np.asarray(list(deleted_rows), dtype=np.int64)] = True
    for lv in range(g["num_levels"] + 1):
        nb = g["level0_neighbors_count"] if lv == 0 else g["neighbors_count"]
        nr = g["node_row"][lv]
        adj = g["adj"][lv].reshape(-1, nb)
        filled = adj != EMPTY
        assert not dead[nr[adj[filled]]].any(), lv              # no slot names a deleted row
        assert not filled[dead[nr]].any(), lv                    # deleted nodes are isolated


ARMS = [(ST.HalfPrecisionFP, MK.Cosine), (ST.UnsignedByte, MK.Cosine), (ST.SubByte2, MK.DotProduct), (ST.HalfPrecisionFP, MK.DotProduct)]


@pytest.mark.parametrize("st,metric", ARMS)
def test_sequential_delete_equals_oracle_after_build_and_after_upload(st, metric):
    n0, dim, levels, nb, nb0, efc, seed = 900, 32, 4, 8, 16, 32, 5
    vecs = clustered(n0, dim, 11)
    zero = st == ST.HalfPrecisionFP and metric == MK.Cosine
    if zero:
        vecs[7] = 0.0   # a zero-norm row: its insert fails (unlinked); deleting it fails its traversal: status 2
    rows = np.concatenate([[7, 7], np.random.default_rng(2).choice(np.arange(8, n0), 80, replace=False), [7]]).astype(np.uint32)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(levels, nb, nb0, efc, 64, 1, seed)
    g0 = ix.read_graph()
    codes, mags = ix.read_codes(0, n0 + 1)
    status = ix.delete_rows(rows, 64, 1)
    o = pydelete.Graph.init(int(metric), int(st), dim, codes, mags, n0, levels, nb, nb0)
    o.insert(0, n0, ef_construction=efc, seed=seed)
    want = o.delete(rows)
    assert np.array_equal(status, want)
    assert status[1] == 1 and status[-1] == 1 and status[0] == (2 if zero else 0)
    assert_graph_equal(ix.read_graph(), o.export(), ix.read_graph_slot_scores(), int(metric))
    assert np.array_equal(np.flatnonzero(ix.deleted_rows()), np.unique(rows))
    # the same deletes on the uploaded first build: slot state derived by hnsw_slot_state_kernel
    up = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 1, keep_raw_f32=True)
    up.append(np.concatenate([vecs, root_vector(seed, dim)[None]]))
    up.set_graph(g0["num_levels"], nb, nb0, g0["entry"], g0["root_row"], g0["node_row"], g0["adj"], g0["child"])
    su = up.delete_rows(rows, 64, 1)
    ou = pydelete.Graph.from_graph(int(metric), int(st), dim, codes, mags, g0)
    assert np.array_equal(su, ou.delete(rows))
    assert_graph_equal(up.read_graph(), ou.export(), up.read_graph_slot_scores(), int(metric))
    for x in (ix, up, o, ou):
        x.close()


def test_update_flow_equals_oracle():
    n0, n1, dim, levels, nb, nb0, efc, seed = 700, 200, 32, 3, 8, 16, 32, 3
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    vecs = clustered(n0 + n1, dim, 17)
    rng = np.random.default_rng(4)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + n1 + 1, keep_raw_f32=True)
    ix.append(vecs[:n0])
    ix.build_graph(levels, nb, nb0, efc, 64, 1, seed)
    codes, mags = ix.read_codes(0, n0 + 1)
    o = pydelete.Graph.init(int(metric), int(st), dim, codes, mags, n0, levels, nb, nb0)
    o.insert(0, n0, ef_construction=efc, seed=seed)
    d1 = rng.choice(n0, 40, replace=False).astype(np.uint32)
    assert np.array_equal(ix.delete_rows(d1, 64, 1), o.delete(d1))
    ix.append(vecs[n0:])
    failed = ix.insert_graph(efc, 64, 1, seed)
    assert failed.size == n1 and failed.sum() == 0
    codes, mags = ix.read_codes(0, n0 + n1 + 1)
    o.set_table(codes, mags)
    assert o.insert(n0 + 1, n1, ef_construction=efc, seed=seed).sum() == 0
    d2 = np.concatenate([rng.choice(np.arange(n0 + 1, n0 + n1 + 1), 20, replace=False), rng.choice(n0, 20, replace=False)]).astype(np.uint32)
    assert np.array_equal(ix.delete_rows(d2, 64, 1), o.delete(d2))
    g = ix.read_graph()
    assert_graph_equal(g, o.export(), ix.read_graph_slot_scores(), int(metric))
    assert_unlinked(g, set(d1.tolist()) | set(d2.tolist()))
    ix.close()
    o.close()


def live_topk(vecs, live, queries, k):
    ids, scores = orc.brute_topk_f32(vecs[live], queries, k)
    return live[ids], scores


def test_batched_delete_invariants_search_parity_and_recall():
    n, dim, k = 20000, 48, 10
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    vecs = clustered(n, dim, 21)
    rng = np.random.default_rng(5)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(5, 16, 32, 64, 64, 4096, 9)
    order = rng.permutation(n).astype(np.uint32)
    raw = np.concatenate([vecs, np.zeros((1, dim), np.float32)])
    queries = (vecs[rng.integers(0, n, 128)] + 0.05 * rng.normal(size=(128, dim))).astype(np.float32)
    done = 0
    for frac in (0.1, 0.5):
        upto = int(n * frac)
        status = ix.delete_rows(order[done:upto])
        assert (status == 0).all()
        done = upto
        dead = order[:done]
        g = ix.read_graph()
        assert_unlinked(g, set(dead.tolist()))
        codes, mags = ix.read_codes(0, n + 1)
        sc = ix.read_graph_slot_scores()
        o = pyinsert.Graph.from_graph(int(metric), int(st), dim, codes, mags, g)   # every similarity recomputed
        e = o.export()
        for lv in range(6):
            filled = g["adj"][lv] != EMPTY
            assert np.array_equal(bits(sc[lv])[filled], bits(pyinsert.slot_scores(int(metric), e["simkey"][lv], e["adj"][lv]))[filled]), lv
        ev0, pp0 = ix.hnsw_counters()
        ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=128, shortlist_size=64)
        ev1, pp1 = ix.hnsw_counters()
        w = o.search_batch(raw, queries, k, ef_search=128)
        o.close()
        assert np.array_equal(ids, w[0]) and np.array_equal(bits(scores), bits(w[1])) and np.array_equal(counts, w[2])
        assert ev1 - ev0 == w[4] and pp1 - pp0 == w[5]
        assert not np.isin(ids, dead).any()
        if frac == 0.1:   # recall@10 against the exact top-10 over the live rows, next to a fresh build over them
            live = np.setdiff1d(np.arange(n), dead)
            gt, _ = live_topk(vecs, live, queries, k)
            rec = np.mean([len(set(ids[i]) & set(gt[i])) / k for i in range(len(queries))])
            fresh = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=live.size + 1, keep_raw_f32=True)
            fresh.append(vecs[live])
            fresh.build_graph(5, 16, 32, 64, 64, 4096, 9)
            fi, _, _, _ = fresh.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=128, shortlist_size=64)
            fresh.close()
            fi = np.where(fi < live.size, live[np.minimum(fi, live.size - 1)], EMPTY)
            rec_fresh = np.mean([len(set(fi[i]) & set(gt[i])) / k for i in range(len(queries))])
            assert rec >= rec_fresh - 0.05, (rec, rec_fresh)
        # the deleted rows' own vectors as queries: no mode returns a deleted row
        q = vecs[dead[:64]]
        for mode in (cdb.SearchMode.HNSW, cdb.SearchMode.BRUTE_RAW, cdb.SearchMode.BRUTE_CODES):
            got, _, _, _ = ix.batch_search(q, k, mode)
            assert not np.isin(got, dead).any(), mode
    ix.close()


@pytest.mark.parametrize("st,mode", [(ST.FullPrecisionFP, cdb.SearchMode.BRUTE_RAW), (ST.UnsignedByte, cdb.SearchMode.BRUTE_CODES)])
def test_brute_force_after_deletes_is_the_exact_scan_over_live_rows(st, mode):
    n, dim, nq, k = 20000, 64, 8, 10
    corpus = orc.synth_matrix(77, n, dim).copy()
    corpus[123] = 0.0   # a zero-norm row: deleted below, it raises no err flag
    q = orc.synth_matrix(78, nq, dim)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=MK.Cosine, capacity=n, keep_raw_f32=st != ST.FullPrecisionFP)
    ix.append(corpus)
    ix.batch_search(q, k, mode)
    assert ix.stats()["tensor_searches"] == 1   # the shape takes a tensor-core path while nothing is deleted
    want_ids, _, _, _ = ix.batch_search(q, k, mode)
    dead = np.unique(np.concatenate([[123], want_ids[:, :3].ravel(), np.random.default_rng(1).choice(n, 2000, replace=False)]))
    assert (ix.delete_rows(dead) == 0).all()
    before = ix.stats()["tensor_searches"]
    ids, scores, counts, err = ix.batch_search(q, k, mode)
    assert ix.stats()["tensor_searches"] == before   # the exact scan answered
    live = np.setdiff1d(np.arange(n), dead)
    if mode == cdb.SearchMode.BRUTE_RAW:
        wi, ws = live_topk(corpus, live, q, k)
        werr = np.zeros(nq, np.uint8)
    else:
        codes, mags = orc.quantize_batch(int(st), corpus)
        qc, qm = orc.quantize_batch(int(st), q)
        rc, wi, ws, werr = orc.brute_topk_codes(int(MK.Cosine), int(st), dim, codes[live], mags[live], qc, qm, k)
        assert rc == 0
        wi = live[wi]
    assert np.array_equal(ids, wi) and np.array_equal(bits(scores), bits(ws))
    assert not err.any() and np.array_equal(err, werr)
    ix.close()


def test_refusals_leave_the_index_unchanged_and_build_insert_skip_deleted_rows():
    n0, dim = 400, 16
    vecs = clustered(n0 + 20, dim, 8)
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.HalfPrecisionFP, metric=MK.Cosine, capacity=n0 + 21, keep_raw_f32=True)
    ix.append(vecs[:n0])
    ix.build_graph(3, 8, 16, 32, 64, 64, 2)
    g0 = ix.read_graph()
    for bad in ([5, n0 + 7], [5, n0]):   # out of range / the root row
        r = np.array(bad, np.uint32)
        rc = ix._lib.cdb_index_delete_rows(ix._h, r.ctypes.data_as(C.c_void_p), r.size, 64, 0, None, None)
        assert rc == int(cdb.Status.INVALID_PARAMS)
    assert not ix.deleted_rows().any()
    g1 = ix.read_graph()
    assert all(np.array_equal(g0["adj"][lv], g1["adj"][lv]) for lv in range(4))
    # a graph naming a deleted row cannot be uploaded
    assert ix.delete_rows([9]).tolist() == [0]
    with pytest.raises(cdb.CosdataError) as e:
        ix.set_graph(g0["num_levels"], 8, 16, g0["entry"], g0["root_row"], g0["node_row"], g0["adj"], g0["child"])
    assert e.value.status == cdb.Status.INVALID_PARAMS
    # a deleted row appended after the build is not inserted (status 2) and not linked
    ix.append(vecs[n0:])
    assert ix.delete_rows([n0 + 5]).tolist() == [0]
    failed = ix.insert_graph(32, 64, 64, 2)
    assert failed.tolist() == [2 if i == 4 else 0 for i in range(20)]
    g = ix.read_graph()
    assert_unlinked(g, {9, n0 + 5})
    ix.close()
    # a build over rows some of which are deleted leaves them out
    b = cdb.DenseIndex(dim=dim, storage_type=ST.HalfPrecisionFP, metric=MK.Cosine, capacity=n0 + 1, keep_raw_f32=True)
    b.append(vecs[:n0])
    assert b.delete_rows([3, 50, 3]).tolist() == [0, 0, 1]
    b.build_graph(3, 8, 16, 32, 64, 64, 2)
    assert_unlinked(b.read_graph(), {3, 50})
    b.close()
    # a graph with metadata: CDB_UNSUPPORTED, nothing marked
    from tests import mdgraph
    pop = mdgraph.replica_population(n=200, dim=16, md_dims=4, levels=2, seed=3)
    nm, dm = pop["vecs"].shape
    m = cdb.DenseIndex(dim=dm, storage_type=ST.HalfPrecisionFP, metric=MK.Cosine, capacity=nm + 3, keep_raw_f32=True)
    m.append(pop["vecs"])
    m.build_graph_replicas(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], pop["md_bits"],
                           pop["md_mags"], pop["main_root_md"], pop["pseudo_root_md"], 2, 8, 16, 16, 64, 64, 1)
    with pytest.raises(cdb.CosdataError) as e:
        m.delete_rows([1])
    assert e.value.status == cdb.Status.UNSUPPORTED and not m.deleted_rows().any()
    m.close()


def test_searches_before_and_after_a_delete_see_the_old_and_the_new_graph():
    import threading
    import torch
    n, dim, k, nq = 5000, 48, 10, 512
    vecs = clustered(n, dim, 31)
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(5, 16, 32, 64, 64, 256, 9)
    old = ix.read_graph()
    rng = np.random.default_rng(6)
    dead = rng.choice(n, 1500, replace=False).astype(np.uint32)
    queries = (vecs[dead[:nq]] + 0.01 * rng.normal(size=(nq, dim))).astype(np.float32)
    dq = torch.from_numpy(queries).cuda()
    out = [(torch.empty((nq, k), dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
            torch.empty(nq, dtype=torch.int32, device="cuda")) for _ in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    enqueued, deleted, errors = threading.Event(), threading.Event(), []

    def searcher():
        try:
            for i in range(2):
                if i == 1:
                    deleted.wait()
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
    status = ix.delete_rows(dead)
    deleted.set()
    t.join()
    assert not errors and (status == 0).all()
    for s_ in streams:
        s_.synchronize()
    new = ix.read_graph()
    codes, mags = ix.read_codes(0, n + 1)
    raw = np.concatenate([vecs, np.zeros((1, dim), np.float32)])
    for graph, (ids, sc, cnt) in zip((old, new), out):
        o = pyinsert.Graph.from_graph(int(metric), int(st), dim, codes, mags, graph)
        w = o.search_batch(raw, queries, k, ef_search=64)
        o.close()
        assert np.array_equal(ids.cpu().numpy().view(np.uint32), w[0])
        assert np.array_equal(bits(sc.cpu().numpy()), bits(w[1])) and np.array_equal(cnt.cpu().numpy().view(np.uint32), w[2])
    assert np.isin(out[0][0].cpu().numpy().view(np.uint32), dead).any()
    assert not np.isin(out[1][0].cpu().numpy().view(np.uint32), dead).any()
    ix.close()
