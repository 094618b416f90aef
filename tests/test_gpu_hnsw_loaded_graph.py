"""Graphs loaded from the reference's index files take inserts and deletes on the GPU (cdb_index_set_graph_slot_scores).
  * cold start of a collection with a metadata schema (prop.data, raw rows, index files, attach): the stored slot values come
    back bit for bit, searches are identical before and after the attach, and one-at-a-time inserts and deletes equal the
    oracle's reload of the same files followed by its insert / delete, failed flags and statuses included;
  * a collection without a metadata schema (no pseudo root) grows and shrinks, searches equal the oracle's on the result,
    and its inserts refuse pseudo replicas and nodes whose Metadata has mag != 0;
  * batched inserts and deletes on a loaded graph keep the replica edge rules, leave no link to a deleted row, search like
    the oracle on the result and keep recall near a one-shot build;
  * refusals leave the index unchanged."""
import ctypes as C
import os

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from oracle import pyhnsw, pymeta
from tests.scored_index_files import METRIC_TAG, LoadedOracle, write_scored_index_dir
from tests.test_gpu_hnsw_insert_replicas import assert_edge_rules, build_a, grown_population, recall, without_nodes

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
EMPTY = 0xFFFFFFFF


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def cold_start(gp, st, metric, levels, nb, nb0, efc, directory, max_batch=1, tag=None):
    """replica build of A on one handle, its index files written with the slot similarities it keeps, then a fresh handle
    cold-started from them as INTEGRATION.md describes (prop.data, raw rows, B appended, index files) -> (source, fresh, files)"""
    n, n_a = gp["n"], gp["n_a"]
    vecs = gp["vecs"]
    dim = vecs.shape[1]
    src, failed = build_a(gp, st, metric, levels, nb, nb0, efc, max_batch)
    assert not failed.any()
    g = src.read_graph()
    ids, mds = src.read_graph_metadata()
    codes, mags = src.read_codes(0, n_a + 2)
    tag = METRIC_TAG[int(metric)] if tag is None else tag
    root_link, pseudo_link = write_scored_index_dir(directory, int(st), dim, codes, mags, g, ids, mds, gp["md_bits"], gp["md_mags"],
                                                    src.read_replica_slot_scores(), tag, pseudo_entry=1, seed=4)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2, keep_raw_f32=True)
    cnt, _ = ix.append_prop_file(os.path.join(directory, "prop.data"))
    assert cnt == n_a + 2
    if st != ST.FullPrecisionFP:                                           # f32 rows are their own raw rows
        ix.set_raw(0, np.concatenate([vecs[:n_a], np.zeros((2, dim), np.float32)]))
    ix.append(vecs[n_a:])
    hf = cdb.HnswFiles(directory, root_link, pseudo_link)
    hf.apply(ix)
    return src, ix, hf


def b_list(gp, n_md_files):
    """B with its Metadata rows renumbered behind the table the files gave (the whole source table is appended once)"""
    b = {c: gp["b"][c].copy() for c in gp["b"]}
    b["md_row"] = np.where(b["md_row"] == EMPTY, EMPTY, b["md_row"] + n_md_files).astype(np.uint32)
    return b, np.concatenate([gp["md_bits"], gp["new_bits"]]), np.concatenate([gp["md_mags"], gp["new_mags"]])


def queries(gp, nq, seed):
    vecs = gp["vecs"]
    rng = np.random.default_rng(seed)
    q = (vecs[rng.integers(0, vecs.shape[0], nq)] + 0.03 * rng.normal(size=(nq, vecs.shape[1]))).astype(np.float32).clip(-0.999, 0.999)
    pats = gp["md_bits"][2:]
    return q, [None if i % 2 == 0 else [pats[i % len(pats)].astype(np.int8)] for i in range(nq)]


def assert_same_graph(ix, e, levels, drop):
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    nbs = [g["level0_neighbors_count"]] + [g["neighbors_count"]] * levels
    got = without_nodes(g["node_row"], ids, mds, g["adj"], g["child"], nbs, drop)
    want = without_nodes(e["node_row"], e["node_id"], e["node_md"], e["adj"], e["child"], nbs, drop)
    for lv in range(levels + 1):
        for key in ("node_row", "node_id", "node_md", "adj") + (("child",) if lv else ()):
            assert np.array_equal(got[key][lv], want[key][lv]), (key, lv)


@pytest.mark.parametrize("st,metric,dim,nb0", [(ST.HalfPrecisionFP, MK.Cosine, 32, 16), (ST.UnsignedByte, MK.Cosine, 32, 16),
                                               (ST.SubByte2, MK.DotProduct, 32, 16), (ST.FullPrecisionFP, MK.Cosine, 32, 16),
                                               (ST.HalfPrecisionFP, MK.Cosine, 768, 64)])
def test_cold_start_insert_and_delete_equal_the_oracle_reload(tmp_path, st, metric, dim, nb0):
    levels, nb, efc = 4, 8, 32
    n, n_a = (500, 300) if dim == 32 else (240, 150)
    gp = grown_population(n, n_a, dim, levels, seed=13, zero=True, pseudo_in_b=True)
    q, filters = queries(gp, 40, 7)
    for calls in (1, 3):
        src, ix, hf = cold_start(gp, st, metric, levels, nb, nb0, efc, str(tmp_path / f"idx{calls}"))
        with pytest.raises(cdb.CosdataError) as e:
            ix.read_replica_slot_scores()
        assert e.value.status == cdb.Status.UNSUPPORTED
        before = ix.batch_search_filtered(q, filters, 5, ef_search=32, shortlist_size=64)
        g0 = ix.read_graph()
        ix.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
        # (a) the stored values come back; (b) searches and the graph are as before
        for lv, s in enumerate(ix.read_replica_slot_scores()):
            assert np.array_equal(bits(s), bits(hf.slot_scores[lv])), lv
        after = ix.batch_search_filtered(q, filters, 5, ef_search=32, shortlist_size=64)
        for x, y in zip(before, after):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
        assert all(np.array_equal(g0["adj"][lv], ix.read_graph()["adj"][lv]) for lv in range(levels + 1))
        # (c) B inserted one node at a time == the oracle's reload + insert
        codes, mags = ix.read_codes(0, n + 2)
        b, tb, tm = b_list(gp, hf.n_md)
        o = LoadedOracle(metric, st, dim, codes, mags, np.concatenate([hf.md_bits, tb]), np.concatenate([hf.md_mags, tm]), levels,
                         nb, nb0, hf.node_row, hf.node_id, hf.node_md, hf.adj, hf.child, hf.slot_scores)
        ofailed = o.insert(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], efc)
        if metric == MK.Cosine:
            assert ofailed[0] == 1                                          # the pseudo replica meets the unreachable arm
        nbn = b["row"].size
        cuts = [0, nbn] if calls == 1 else [0, nbn // 3, 2 * nbn // 3, nbn]
        fb = []
        for c in range(len(cuts) - 1):
            lo, hi = cuts[c], cuts[c + 1]
            kw = dict(md_bits_new=tb, md_mags_new=tm) if c == 0 else {}
            fb.append(ix.insert_graph_replicas(b["row"][lo:hi], b["node_id"][lo:hi], b["base_id"][lo:hi], b["md_row"][lo:hi],
                                               b["max_level"][lo:hi], ef_construction=efc, shortlist_size=64, max_batch=1, **kw))
        fb = np.concatenate(fb)
        assert np.array_equal(fb, ofailed), calls
        drop = b["node_id"][ofailed != 0]
        assert_same_graph(ix, o.export(), levels, drop)
        # (d) then rows deleted one at a time == the oracle's delete on the same state
        rng = np.random.default_rng(calls)
        rows = np.concatenate([rng.choice(n_a, 8, replace=False), n_a + 2 + rng.choice(n - n_a, 6, replace=False)]).astype(np.uint32)
        got = ix.delete_rows_replicas(rows, 64, 1)
        want = o.delete(rows)
        assert np.array_equal(got, want)
        assert_same_graph(ix, o.export(), levels, drop)
        o.close(); hf.close(); ix.close(); src.close()


def graph_scores_equal(ix, e, levels, metric):
    """the GPU graph == an oracle export (same numbering): node_row, adj, child and every filled slot's similarity"""
    from tests import pyinsert
    g = ix.read_graph()
    sc = ix.read_replica_slot_scores()
    for lv in range(levels + 1):
        for key in ("node_row", "adj") + (("child",) if lv else ()):
            assert np.array_equal(g[key][lv], e[key][lv]), (key, lv)
        assert np.array_equal(bits(sc[lv]), bits(pyinsert.slot_scores(int(metric), e["simkey"][lv], e["adj"][lv]))), lv


@pytest.mark.parametrize("ids_are_rows", [True, False])
def test_collection_without_a_schema(tmp_path, ids_are_rows):
    """no metadata schema, so no pseudo root.  One node at a time, inserts and deletes on the graph cold-started from the files
    equal the oracle's reload of those files (no pseudo root).  With prop ids = rows they also equal the plain insert and
    delete oracles on the source graph (the same graph uploaded in the plain numbering); with other ids, search on the
    grown graph equals the oracle's, whose fixed set is keyed by those ids."""
    from tests import pydelete
    levels, nb, nb0, efc, k = 3, 8, 16, 48, 10
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 32
    n_a, n_b = 1500, 400
    vecs = orc.synth_matrix(77, n_a + n_b, dim)
    src = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n_a + 1, keep_raw_f32=True)
    src.append(vecs[:n_a])
    src.build_graph(levels, nb, nb0, efc, 64, 1, 3)
    g = src.read_graph()
    scores = src.read_graph_slot_scores()
    codes, mags = src.read_codes(0, n_a + 1)
    src.close()
    prop_id = np.arange(n_a + 1 + n_b, dtype=np.uint32) if ids_are_rows else (np.arange(n_a + 1 + n_b) * 4 + 1).astype(np.uint32)
    prop_id[n_a] = EMPTY                                                    # the root's id is u32::MAX
    ids = [prop_id[a] for a in g["node_row"]]
    mds = [np.full(a.size, EMPTY, np.uint32) for a in g["node_row"]]
    d = str(tmp_path / "plain")
    root_link, _ = write_scored_index_dir(d, int(st), dim, codes, mags, g, ids, mds, np.zeros((0, 1), np.int32), np.zeros(0, np.float32),
                                          scores, METRIC_TAG[int(metric)], row_ids=prop_id)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n_a + 1 + n_b, keep_raw_f32=True)
    ix.append_prop_file(os.path.join(d, "prop.data"))
    ix.set_raw(0, np.concatenate([vecs[:n_a], np.zeros((1, dim), np.float32)]))
    ix.append(vecs[n_a:])
    hf = cdb.HnswFiles(d, root_link)
    assert hf.pseudo_entry == EMPTY
    hf.apply(ix, slot_scores=True)
    for lv, s in enumerate(ix.read_replica_slot_scores()):
        assert np.array_equal(bits(s), bits(hf.slot_scores[lv])), lv
    # refusals of a graph without a pseudo root: nothing changes
    g0 = ix.read_graph()
    rows = np.arange(n_a + 1, n_a + 1 + n_b, dtype=np.uint32)
    new_ids = prop_id[rows]
    draws = np.random.default_rng(1).integers(0, 3, n_b).astype(np.uint8)
    for row, md_row, new in ((EMPTY, EMPTY, None), (rows[0], 0, (np.ones((1, 1), np.int32), np.ones(1, np.float32)))):
        with pytest.raises(cdb.CosdataError) as e:
            ix.insert_graph_replicas([row], [7], [7], [md_row], [0], *(new or (None, None)), efc, 64, 64)
        assert e.value.status == cdb.Status.INVALID_PARAMS and "no pseudo root" in str(e.value)
    with pytest.raises(cdb.CosdataError) as e:
        ix.delete_rows_replicas([g0["root_row"]])
    assert e.value.status == cdb.Status.INVALID_PARAMS
    assert all(np.array_equal(g0["adj"][lv], ix.read_graph()["adj"][lv]) for lv in range(levels + 1))
    # one node at a time: B inserted, then rows deleted == the oracle's reload of the files (no pseudo root)
    codes, mags = ix.read_codes(0, n_a + 1 + n_b)
    o = LoadedOracle(metric, st, dim, codes, mags, np.zeros((1, 1), np.int32), np.zeros(1, np.float32), levels, nb, nb0, hf.node_row,
                     hf.node_id, hf.node_md, hf.adj, hf.child, hf.slot_scores, entry=hf.entry, pseudo_entry=None)
    no_md = np.full(n_b, EMPTY, np.uint32)
    fb = ix.insert_graph_replicas(rows, new_ids, new_ids, no_md, draws, None, None, efc, 64, 1)
    assert np.array_equal(fb, o.insert(rows, new_ids, new_ids, no_md, draws, efc)) and fb.sum() == 0
    e = o.export()
    gids, _ = ix.read_graph_metadata()
    assert all(np.array_equal(gids[lv], e["node_id"][lv]) for lv in range(levels + 1))
    graph_scores_equal(ix, e, levels, metric)
    rng = np.random.default_rng(2)
    dead = rng.choice(np.concatenate([np.arange(n_a), rows]), 120, replace=False).astype(np.uint32)
    dead = np.concatenate([dead, dead[:3]])                                 # already deleted: status 1
    got = ix.delete_rows_replicas(dead, 64, 1)
    assert np.array_equal(got, o.delete(dead)) and (got[-3:] == 1).all()
    graph_scores_equal(ix, o.export(), levels, metric)
    o.close()
    if ids_are_rows:
        # the plain oracles (ig_from_graph + ig_insert_rows, the plain delete) on the source graph; the GPU side is the same
        # graph uploaded in the plain numbering with the stored similarities attached
        up = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n_a + 1 + n_b, keep_raw_f32=True)
        up.append_codes(codes, mags)
        up.set_raw(0, np.concatenate([vecs[:n_a], np.zeros((1, dim), np.float32), vecs[n_a:]]))
        up.set_graph(g["num_levels"], nb, nb0, g["entry"], g["root_row"], g["node_row"], g["adj"], g["child"])
        up.set_graph_metadata(np.zeros((1, 1), np.int32), np.zeros(1, np.float32), ids, mds, g["entry"])
        up.set_graph_slot_scores(scores)
        q = pydelete.Graph.from_graph(int(metric), int(st), dim, codes, mags, g)
        fu = up.insert_graph_replicas(rows, new_ids, new_ids, no_md, draws, None, None, efc, 64, 1)
        assert np.array_equal(fu, q.insert(n_a + 1, n_b, ef_construction=efc, max_level=draws))
        graph_scores_equal(up, q.export(), levels, metric)
        assert np.array_equal(up.delete_rows_replicas(dead, 64, 1), q.delete(dead))
        graph_scores_equal(up, q.export(), levels, metric)
        q.close(); up.close()
    # search on the grown and shrunk graph == the oracle's (the fixed set keyed by the node ids)
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    nq = 60
    qv = (vecs[rng.integers(0, n_a + n_b, nq)] + 0.03 * rng.normal(size=(nq, dim))).astype(np.float32).clip(-0.999, 0.999)
    fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n_a, levels, nb, nb0, g["entry"], g["node_row"], g["adj"], g["child"])
    mg = pymeta.MdGraph(fg, np.zeros((1, 1), np.int32), np.zeros(1, np.float32), ids, mds, g["entry"])
    raw = np.concatenate([vecs[:n_a], np.zeros((1, dim), np.float32), vecs[n_a:]])
    r_ids, r_sc, r_cnt, r_err = ix.batch_search_filtered(qv, [None] * nq, k, ef_search=64, shortlist_size=64)
    w = pymeta.search_batch_md(mg, raw, qv, [None] * nq, k, ef_search=64)
    assert np.array_equal(r_err, w[3]) and np.array_equal(r_cnt, w[2])
    assert np.array_equal(r_ids, w[0]) and np.array_equal(bits(r_sc), bits(w[1]))
    assert not np.isin(r_ids, prop_id[dead]).any() and r_cnt.min() > 0
    hf.close(); ix.close()


def test_batched_inserts_and_deletes_on_a_loaded_graph(tmp_path):
    levels, nb, nb0, efc, k = 5, 16, 32, 64, 10
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 48
    n, n_a = 6000, 4000
    gp = grown_population(n, n_a, dim, levels, seed=17, chunks=10)
    vecs = gp["vecs"]
    src, ix, hf = cold_start(gp, st, metric, levels, nb, nb0, efc, str(tmp_path / "idx"), max_batch=256)
    src.close()
    ix.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
    b, tb, tm = b_list(gp, hf.n_md)
    failed = ix.insert_graph_replicas(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], tb, tm, efc, 64, 4096)
    assert failed.sum() == 0
    rng = np.random.default_rng(3)
    data_rows = np.concatenate([np.arange(n_a), n_a + 2 + np.arange(n - n_a)])
    dead = rng.choice(data_rows, n // 10, replace=False).astype(np.uint32)
    assert (ix.delete_rows_replicas(dead, 64, 4096) != 1).all()
    md_bits, md_mags = np.concatenate([hf.md_bits, tb]), np.concatenate([hf.md_mags, tm])
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    assert_edge_rules(g, ids, mds, md_bits, md_mags, levels, nb, nb0)
    dead_set = np.zeros(n + 2, bool)
    dead_set[dead] = True
    for lv in range(levels + 1):
        a = g["adj"][lv]
        assert not dead_set[g["node_row"][lv][a[a != EMPTY]]].any(), lv
    # CUDA search == the oracle's on the resulting graph; recall near a one-shot build over the live rows
    nq = 80
    q, filters = queries(gp, nq, 9)
    codes, mags = ix.read_codes(0, n + 2)
    fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n_a, levels, nb, nb0, g["entry"], g["node_row"], g["adj"], g["child"])
    mg = pymeta.MdGraph(fg, md_bits, md_mags, ids, mds, hf.pseudo_entry)
    raw = np.concatenate([vecs[:n_a], np.zeros((2, dim), np.float32), vecs[n_a:]])
    r = ix.batch_search_filtered(q, filters, k, ef_search=64, shortlist_size=64)
    w = pymeta.search_batch_md(mg, raw, q, filters, k, ef_search=64)
    for x, y in zip(r, w):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    live = np.setdiff1d(np.arange(n), np.where(dead >= n_a + 2, dead - 2, dead))
    unf = [i for i in range(nq) if filters[i] is None]
    gt = np.zeros((len(unf), k), np.int64)
    for j, i in enumerate(unf):
        ids_, _ = orc.brute_topk_f32(vecs[live], q[i:i + 1], k)
        gt[j] = live[ids_[0]]
    one = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2, keep_raw_f32=True)
    one.append(vecs)
    a_, b_ = gp["a"], gp["b"]
    all_rows = np.concatenate([a_["row"], np.where(b_["row"] == EMPTY, EMPTY, b_["row"] - 2)]).astype(np.uint32)
    keep = (all_rows == EMPTY) | np.isin(all_rows, live)
    all_md = np.concatenate([a_["md_row"], gp["b"]["md_row"]])
    one.build_graph_replicas(all_rows[keep], np.concatenate([a_["node_id"], b_["node_id"]])[keep],
                             np.concatenate([a_["base_id"], b_["base_id"]])[keep], all_md[keep],
                             np.concatenate([a_["max_level"], b_["max_level"]])[keep], np.concatenate([gp["md_bits"], gp["new_bits"]]),
                             np.concatenate([gp["md_mags"], gp["new_mags"]]), gp["main_root_md"], gp["pseudo_root_md"],
                             levels, nb, nb0, efc, 64, 256, 1)
    i1, _, c1, _ = one.batch_search_filtered(q[unf], [None] * len(unf), k, ef_search=64, shortlist_size=64)
    one.close()
    r_ids, r_counts = r[0][unf], r[2][unf]
    rec_loaded = recall(r_ids, r_counts, gt, k)
    rec_one = recall(i1, c1, gt, k)
    assert rec_loaded >= rec_one - 0.05, (rec_loaded, rec_one)
    hf.close(); ix.close()


def test_refusals_leave_the_index_unchanged(tmp_path):
    levels, nb, nb0, efc = 3, 8, 16, 16
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 24
    gp = grown_population(300, 200, dim, levels, seed=5)
    INV, MIS, UNS = cdb.Status.INVALID_PARAMS, cdb.Status.STORAGE_MISMATCH, cdb.Status.UNSUPPORTED
    lib = cdb._lib.load()
    # no graph, and a graph without metadata
    plain = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=400, keep_raw_f32=True)
    plain.append(gp["vecs"])
    t = (C.c_void_p * 1)(None)
    assert lib.cdb_index_set_graph_slot_scores(plain._h, C.cast(t, C.c_void_p), None) == INV
    plain.build_graph(levels, nb, nb0, efc, 64, 64, 1)
    g = plain.read_graph()
    with pytest.raises(cdb.CosdataError) as e:
        plain.set_graph_slot_scores(plain.read_graph_slot_scores())
    assert e.value.status == INV
    assert np.array_equal(plain.read_graph()["adj"][0], g["adj"][0])
    plain.close()
    # tags of another metric (DotProductDistance under cosine): CDB_STORAGE_MISMATCH, the graph stays read-only
    src, ix, hf = cold_start(gp, st, metric, levels, nb, nb0, efc, str(tmp_path / "dot"), max_batch=64, tag=4)
    src.close()
    q, filters = queries(gp, 20, 3)
    s0 = ix.batch_search_filtered(q, filters, 5, ef_search=32)
    g0 = ix.read_graph()
    with pytest.raises(cdb.CosdataError) as e:
        ix.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
    assert e.value.status == MIS
    s1 = ix.batch_search_filtered(q, filters, 5, ef_search=32)
    for x, y in zip(s0, s1):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    assert all(np.array_equal(g0[key][lv], ix.read_graph()[key][lv]) for key in ("node_row", "adj") for lv in range(levels + 1))
    for call in (ix.read_replica_slot_scores, lambda: ix.delete_rows_replicas([0])):
        with pytest.raises(cdb.CosdataError) as e:
            call()
        assert e.value.status == UNS
    ix.set_graph_slot_scores(hf.slot_scores)                               # without tags nothing is checked
    hf.close(); ix.close()
    src, ix, hf = cold_start(gp, st, metric, levels, nb, nb0, efc, str(tmp_path / "ok"), max_batch=64)
    src.close()
    s0 = ix.batch_search_filtered(q, filters, 5, ef_search=32)
    g0 = ix.read_graph()
    bad_tags = [t.copy() for t in hf.slot_tags]
    bad_tags[0][np.flatnonzero(hf.adj[0] != EMPTY)[-1]] = 2
    cases = [(dict(scores=hf.slot_scores, tags=bad_tags), MIS),
             (dict(scores=hf.slot_scores[:-1]), ValueError),
             (dict(scores=[s[:-1] for s in hf.slot_scores]), ValueError)]
    for kw, want in cases:
        with pytest.raises((cdb.CosdataError, ValueError)) as e:
            ix.set_graph_slot_scores(**kw)
        assert (e.type is ValueError) if want is ValueError else e.value.status == want
    t = (C.c_void_p * (levels + 1))(*([hf.slot_scores[0].ctypes.data] + [None] * levels))
    assert lib.cdb_index_set_graph_slot_scores(ix._h, C.cast(t, C.c_void_p), None) == INV
    # a level listing a node id twice
    ids = [a.copy() for a in hf.node_id]
    ids[0][5] = ids[0][6]
    dup = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=gp["n"] + 2, keep_raw_f32=True)
    codes, mags = ix.read_codes(0, gp["n"] + 2)
    dup.append_codes(codes, mags)
    dup.set_raw(0, np.concatenate([gp["vecs"][:gp["n_a"]], np.zeros((2, dim), np.float32), gp["vecs"][gp["n_a"]:]]))
    dup.set_graph(hf.num_levels, nb, nb0, hf.entry, hf.root_row, hf.node_row, hf.adj, hf.child)
    dup.set_graph_metadata(hf.md_bits, hf.md_mags, ids, hf.node_md, hf.pseudo_entry)
    with pytest.raises(cdb.CosdataError) as e:
        dup.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
    assert e.value.status == INV and "twice" in str(e.value)
    with pytest.raises(cdb.CosdataError) as e:
        dup.read_replica_slot_scores()
    assert e.value.status == UNS
    dup.close()
    # every refusal left the graph, its searches and its read-only state as they were
    s1 = ix.batch_search_filtered(q, filters, 5, ef_search=32)
    for x, y in zip(s0, s1):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    assert all(np.array_equal(g0[key][lv], ix.read_graph()[key][lv]) for key in ("node_row", "adj") for lv in range(levels + 1))
    with pytest.raises(cdb.CosdataError) as e:
        ix.delete_rows_replicas([0])
    assert e.value.status == UNS
    # attached once; a second attach is refused
    ix.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
    with pytest.raises(cdb.CosdataError) as e:
        ix.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
    assert e.value.status == INV
    hf.close(); ix.close()


def test_a_search_enqueued_before_the_attach_sees_the_old_state(tmp_path):
    import threading
    import torch
    levels, nb, nb0, efc, k, nq = 5, 16, 32, 64, 10, 256
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 48
    n, n_a = 5000, 4000
    gp = grown_population(n, n_a, dim, levels, seed=31)
    vecs = gp["vecs"]
    src, ix, hf = cold_start(gp, st, metric, levels, nb, nb0, efc, str(tmp_path / "idx"), max_batch=256)
    src.close()
    old_g = ix.read_graph()
    old_ids, old_mds = ix.read_graph_metadata()
    rng = np.random.default_rng(6)
    queries_ = (vecs[rng.integers(n_a, n, nq)] + 0.03 * rng.normal(size=(nq, dim))).astype(np.float32).clip(-0.999, 0.999)
    dq = torch.from_numpy(queries_).cuda()
    out = [(torch.empty((nq, k), dtype=torch.int32, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"),
            torch.empty(nq, dtype=torch.int32, device="cuda")) for _ in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    enqueued, written, errors = threading.Event(), threading.Event(), []

    def searcher():
        try:
            for i in range(2):
                if i == 1:
                    written.wait()
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
    ix.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
    b, tb, tm = b_list(gp, hf.n_md)
    failed = ix.insert_graph_replicas(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], tb, tm, efc, 64, 256)
    written.set()
    t.join()
    assert not errors and failed.sum() == 0
    for s_ in streams:
        s_.synchronize()
    new_g = ix.read_graph()
    new_ids, new_mds = ix.read_graph_metadata()
    codes, mags = ix.read_codes(0, n + 2)
    raw = np.concatenate([vecs[:n_a], np.zeros((2, dim), np.float32), vecs[n_a:]])
    tables = ((hf.md_bits, hf.md_mags), (np.concatenate([hf.md_bits, tb]), np.concatenate([hf.md_mags, tm])))
    for (g, ids_, mds_), (tbits, tmags), (r_ids, r_sc, r_cnt) in zip(((old_g, old_ids, old_mds), (new_g, new_ids, new_mds)), tables, out):
        fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n_a, levels, nb, nb0, g["entry"], g["node_row"], g["adj"], g["child"])
        mg = pymeta.MdGraph(fg, tbits, tmags, ids_, mds_, hf.pseudo_entry)
        w = pymeta.search_batch_md(mg, raw, queries_, [None] * nq, k, ef_search=64)
        assert np.array_equal(r_ids.cpu().numpy().view(np.uint32), w[0])
        assert np.array_equal(bits(r_sc.cpu().numpy()), bits(w[1])) and np.array_equal(r_cnt.cpu().numpy().view(np.uint32), w[2])
    new_set = set(b["node_id"].tolist())
    got = [set(x.cpu().numpy().view(np.uint32).ravel().tolist()) for x in (out[0][0], out[1][0])]
    assert not (got[0] & new_set) and (got[1] & new_set)
    hf.close(); ix.close()
