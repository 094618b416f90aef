"""cdb_index_delete_rows_replicas: deleting embeddings from a graph with metadata (replica graph) on the GPU.
  * one row at a time, the result equals the replica delete oracle (tests/hnsw_delete_md_oracle.c) array for array: node
    rows, ids, Metadata rows, adjacency, children, slot scores and statuses, after a build and through build / delete /
    insert / delete;
  * batched deletes leave no link to a deleted row's nodes, keep the edge rules and every slot similarity exact, search
    equals the oracle's on the repaired graph, and recall stays near a fresh build over the live embeddings;
  * a deleted embedding never comes back, from HNSW (filtered or not) or the exact scans;
  * refusals leave the index unchanged, and a search enqueued before a delete sees the old graph."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from oracle import pyhnsw, pymeta
from tests import mdgraph, pydelete_md
from tests.test_gpu_hnsw_insert_replicas import (assert_edge_rules, build_a, full_table, grown_population, insert_b,
                                                 without_nodes)

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
EMPTY = 0xFFFFFFFF


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def gpu_index(pop, vecs, st, metric, levels, nb, nb0, efc, max_batch, extra=0):
    n, dim = vecs.shape
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2 + extra, keep_raw_f32=True)
    ix.append(vecs)
    failed = ix.build_graph_replicas(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], pop["md_bits"],
                                     pop["md_mags"], pop["main_root_md"], pop["pseudo_root_md"], levels, nb, nb0, efc, 64, max_batch, 1)
    return ix, failed


def oracle_for(ix, st, metric, dim, md_bits, md_mags, levels, nb, nb0, main_root_row, main_root_md, pseudo_root_md, rows_total):
    codes, mags = ix.read_codes(0, rows_total)
    return pydelete_md.Graph(metric, st, dim, codes, mags, md_bits, md_mags, levels, nb, nb0, main_root_row, main_root_md,
                             main_root_row + 1, pseudo_root_md)


def assert_equal_to_oracle(ix, og, levels, metric, drop_ids):
    """GPU graph == oracle graph array for array (slot scores as order keys).  Entries whose insert failed keep isolated
    nodes on different levels on the two sides (see test_gpu_hnsw_insert_replicas): both are compared without them."""
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    sc = ix.read_replica_slot_scores()
    e = og.export()
    nbs = [g["level0_neighbors_count"]] + [g["neighbors_count"]] * levels
    drop = np.array(sorted(drop_ids), np.uint32)
    got = without_nodes(g["node_row"], ids, mds, g["adj"], g["child"], nbs, drop)
    want = without_nodes(e["node_row"], e["node_id"], e["node_md"], e["adj"], e["child"], nbs, drop)
    for lv in range(levels + 1):
        for key in ("node_row", "node_id", "node_md", "adj") + (("child",) if lv else ()):
            assert np.array_equal(got[key][lv], want[key][lv]), (key, lv)
        kg, kw = ~np.isin(ids[lv], drop), ~np.isin(e["node_id"][lv], drop)
        filled = g["adj"][lv].reshape(-1, nbs[lv])[kg] != EMPTY
        got_keys = pydelete_md.order_keys(metric, sc[lv].reshape(-1, nbs[lv])[kg][filled])
        assert np.array_equal(got_keys, e["simkey"][lv].reshape(-1, nbs[lv])[kw][filled]), ("slot scores", lv)


def no_links_to_deleted(ix, deleted_rows, levels):
    g = ix.read_graph()
    dead = np.zeros(len(ix), bool)
    dead[np.asarray(list(deleted_rows), np.int64)] = True
    for lv in range(levels + 1):
        nb = g["level0_neighbors_count"] if lv == 0 else g["neighbors_count"]
        adj = g["adj"][lv].reshape(-1, nb)
        nr = g["node_row"][lv].astype(np.int64)
        is_dead = dead[nr]
        is_dead[:2] = False
        assert (adj[is_dead] == EMPTY).all(), lv                             # every deleted node is isolated
        named = adj[adj != EMPTY]
        assert not is_dead[named].any(), lv                                  # no slot names a deleted node


def pick(pop, n, rng, count, exclude=()):
    """rows with only a base replica, with one and with two Metadata replicas"""
    reps = np.bincount(pop["row"][pop["row"] != EMPTY], minlength=n)
    out = []
    for c in (1, 2, 3):
        grp = np.setdiff1d(np.flatnonzero(reps == c), np.asarray(list(exclude), np.int64))
        out.append(rng.choice(grp, count // 3, replace=False))
    return np.concatenate(out)


@pytest.mark.parametrize("st,metric,dim,nb0", [(ST.HalfPrecisionFP, MK.Cosine, 32, 16), (ST.UnsignedByte, MK.Cosine, 32, 16),
                                               (ST.SubByte2, MK.DotProduct, 32, 16), (ST.FullPrecisionFP, MK.Cosine, 32, 16),
                                               (ST.HalfPrecisionFP, MK.Cosine, 768, 64)])
def test_sequential_delete_equals_oracle(st, metric, dim, nb0):
    levels, nb, efc = 4, 8, 32
    n = 400 if dim == 32 else 200
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=23)
    reps = np.bincount(pop["row"][pop["row"] != EMPTY], minlength=n)
    zero = int(np.flatnonzero(reps == 3)[1])
    vecs = pop["vecs"].copy()
    vecs[zero] = 0.0
    ix, failed = gpu_index(pop, vecs, st, metric, levels, nb, nb0, efc, 1, extra=3)
    ix.append(mdgraph.replica_population(n=3, dim=dim, seed=5)["vecs"])   # rows n+2.. are never listed: only marked
    og = oracle_for(ix, st, metric, dim, pop["md_bits"], pop["md_mags"], levels, nb, nb0, n, pop["main_root_md"], pop["pseudo_root_md"],
                    n + 5)
    ofailed = og.insert(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], efc)
    assert np.array_equal(failed, ofailed)
    drop = set(pop["node_id"][failed != 0].tolist())
    rng = np.random.default_rng(7)
    rows1 = list(pick(pop, n, rng, 48, exclude=[zero])) + [zero, n + 3]
    rows1 = [int(r) for r in rng.permutation(rows1)]
    rows1.insert(5, rows1[2])                                            # a duplicate: status 1
    s = ix.delete_rows_replicas(rows1, max_batch=1)
    w = og.delete(rows1)
    assert np.array_equal(s, w) and s[5] == 1
    if metric == MK.Cosine and st in (ST.HalfPrecisionFP, ST.FullPrecisionFP):
        assert s[rows1.index(zero)] == 2                                 # the zero-norm row's traversals fail
    assert_equal_to_oracle(ix, og, levels, int(metric), drop)
    rows2 = [rows1[0]] + [int(r) for r in pick(pop, n, rng, 9, exclude=rows1)]
    s = ix.delete_rows_replicas(rows2, max_batch=1)
    w = og.delete(rows2)
    assert np.array_equal(s, w) and s[0] == 1                            # deleted by the earlier call
    assert_equal_to_oracle(ix, og, levels, int(metric), drop)
    assert np.array_equal(np.flatnonzero(ix.deleted_rows()), np.flatnonzero(og.deleted[: n + 5]))
    no_links_to_deleted(ix, set(rows1 + rows2), levels)
    ix.close()
    og.close()


@pytest.mark.parametrize("st", [ST.HalfPrecisionFP, ST.UnsignedByte, ST.FullPrecisionFP])
def test_sequential_replica_relinks_equal_oracle(st):
    """small neighbour lists (2 levels, 4 / 8 neighbours) where D5's relinks run: deleting the first embeddings with Metadata
    replicas empties pseudo nodes (a Pseudo node rescoring a Metadata candidate: the unreachable arm, status 2), and
    Metadata and Base nodes empty and are relinked with the replica arms and the edge rules.  The two Metadata replicas of
    a row carry twin patterns, so they share neighbours and the list-order repair decides which candidates a shared
    neighbour is relinked from.  The oracle is itself checked against the Python restatement on the same deletes."""
    from tests.test_oracle_hnsw_delete_md import PyMd, early_and_more_metadata_rows, twin_population
    levels, nb, nb0, efc, metric, dim, n = 2, 4, 8, 32, MK.Cosine, 32, 400
    pop = twin_population(n, dim, levels)
    ix, failed = gpu_index(pop, pop["vecs"], st, metric, levels, nb, nb0, efc, 1)
    og = oracle_for(ix, st, metric, dim, pop["md_bits"], pop["md_mags"], levels, nb, nb0, n, pop["main_root_md"], pop["pseudo_root_md"],
                    n + 2)
    assert np.array_equal(failed, og.insert(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], efc))
    assert not failed.any()
    rows = early_and_more_metadata_rows(pop, n, 230)
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    adj0, nr0 = g["adj"][0].reshape(-1, nb0), g["node_row"][0]
    shared = 0   # deleted rows whose two Metadata replicas share a level-0 neighbour: their repair order matters
    for r in rows:
        a = np.flatnonzero((nr0 == r) & (mds[0] != EMPTY) & (mds[0] >= 2))
        if a.size == 2:
            na, nb_ = (set(adj0[x][adj0[x] != EMPTY].tolist()) for x in a)
            shared += bool(na & nb_)
    assert shared > 10
    row = np.where(pop["row"] == EMPTY, n + 1, pop["row"])
    p = PyMd(og.export(), og, list(zip(row.tolist(), pop["node_id"].tolist(), pop["md_row"].tolist())))
    pdel = og.deleted.copy()
    want = np.array([p.delete(int(r), pdel, 64) for r in rows], np.uint8)
    assert p.relinks > 20 and p.rule_skips > 0 and p.unreachable > 0   # the paths this test is about did run
    w = og.delete(rows)
    assert np.array_equal(w, want)
    s = ix.delete_rows_replicas(rows, max_batch=1)
    assert np.array_equal(s, w) and (s == 2).sum() == p.unreachable    # status 2 from relink Errs only
    assert_equal_to_oracle(ix, og, levels, int(metric), ())
    no_links_to_deleted(ix, set(rows), levels)
    ix.close()
    og.close()


def test_build_delete_insert_delete_equals_oracle():
    levels, nb, nb0, efc = 4, 8, 16, 32
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 32
    gp = grown_population(500, 300, dim, levels, seed=29, chunks=1)
    n, n_a = gp["n"], gp["n_a"]
    ix, fa = build_a(gp, st, metric, levels, nb, nb0, efc, 1)
    md_bits, md_mags = full_table(gp)
    og = oracle_for(ix, st, metric, dim, md_bits, md_mags, levels, nb, nb0, n_a, gp["main_root_md"], gp["pseudo_root_md"], n + 2)
    a, b = gp["a"], gp["b"]
    assert np.array_equal(fa, og.insert(a["row"], a["node_id"], a["base_id"], a["md_row"], a["max_level"], efc))
    rng = np.random.default_rng(3)
    rows1 = [int(r) for r in rng.choice(n_a, 30, replace=False)]
    assert np.array_equal(ix.delete_rows_replicas(rows1, max_batch=1), og.delete(rows1))
    fb = insert_b(ix, gp, efc, 1, 1)
    assert np.array_equal(fb, og.insert(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], efc))
    b_rows = np.unique(b["row"][b["row"] != EMPTY])
    rows2 = [int(r) for r in rng.choice(np.setdiff1d(np.arange(n_a), rows1), 15, replace=False)] + \
            [int(r) for r in rng.choice(b_rows, 15, replace=False)] + [rows1[3]]
    rows2 = [int(r) for r in rng.permutation(rows2)]
    s = ix.delete_rows_replicas(rows2, max_batch=1)
    assert np.array_equal(s, og.delete(rows2)) and (s == 1).sum() == 1
    all_ids = np.concatenate([a["node_id"], b["node_id"]])
    assert_equal_to_oracle(ix, og, levels, int(metric), set(all_ids[np.concatenate([fa, fb]) != 0].tolist()))
    no_links_to_deleted(ix, set(rows1 + rows2), levels)
    ix.close()
    og.close()


def slot_scores_exact(ix, md_bits, md_mags, levels, metric, st):
    """every filled slot: the stored similarity == calculate(x, y) recomputed by the oracle, x the Metadata end of a
    Pseudo-Metadata edge (those arms are not symmetric)"""
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    sc = ix.read_replica_slot_scores()
    codes, mags = ix.read_codes(0, len(ix))
    fg = pyhnsw.FlatGraph(int(metric), int(st), ix.dim, codes, mags, g["root_row"], levels, g["neighbors_count"],
                          g["level0_neighbors_count"], g["entry"], g["node_row"], g["adj"], g["child"])
    mg = pymeta.MdGraph(fg, md_bits, md_mags, ids, mds, 1)
    for lv in range(levels + 1):
        want, rc = pydelete_md.slot_calc(mg, lv)
        filled = g["adj"][lv] != EMPTY
        assert filled.any() and (rc[filled] == 0).all() and (rc[~filled] == -1).all(), lv
        assert np.array_equal(bits(sc[lv][filled]), bits(want[filled])), lv


def live_recall(vecs, pop, deleted, q, filters, r_ids, r_counts, k, id_row):
    live = np.setdiff1d(np.arange(vecs.shape[0]), np.asarray(sorted(deleted), np.int64))
    gt = np.full((len(q), k), -1, np.int64)
    for i in range(len(q)):
        if filters[i] is None:
            cand = live
        else:
            carries = (pop["md_row"] != EMPTY) & (pop["row"] != EMPTY) & \
                      (pop["md_bits"][np.minimum(pop["md_row"], pop["md_bits"].shape[0] - 1)] == filters[i][0]).all(1)
            cand = np.intersect1d(np.unique(pop["row"][carries]), live)
        ids_, _ = orc.brute_topk_f32(vecs[cand], q[i:i + 1], min(k, cand.size))
        gt[i, : ids_.shape[1]] = cand[ids_[0]]
    rows = np.vectorize(lambda x: id_row.get(int(x), -2))(r_ids)
    return np.mean([len(set(rows[i, : r_counts[i]].tolist()) & set(gt[i][gt[i] >= 0].tolist())) / k for i in range(len(q))])


def test_batched_deletes_keep_the_invariants():
    levels, nb, nb0, efc, k = 5, 16, 32, 64, 10
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 48
    n = 6000
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=37)
    vecs = pop["vecs"]
    id_row = {int(i): int(r) for i, r in zip(pop["node_id"], pop["row"]) if r != EMPTY}
    ix, failed = gpu_index(pop, vecs, st, metric, levels, nb, nb0, efc, 256)
    assert failed.sum() == 0
    rng = np.random.default_rng(8)
    nq = 90
    q = (vecs[rng.integers(0, n, nq)] + 0.03 * rng.normal(size=(nq, dim))).astype(np.float32).clip(-0.999, 0.999)
    pats = pop["md_bits"][2:]
    filters = [None if i % 2 == 0 else [pats[i % len(pats)].astype(np.int8)] for i in range(nq)]
    raw = np.concatenate([vecs, np.zeros((2, dim), np.float32)])
    order = rng.permutation(n)
    deleted = set()
    for frac in (0.1, 0.5):
        rows = [int(r) for r in order[len(deleted):int(frac * n)]]
        s = ix.delete_rows_replicas(rows)
        assert (s != 1).all()
        deleted.update(rows)
        assert ix.deleted_rows().sum() == len(deleted)
        no_links_to_deleted(ix, deleted, levels)
        g = ix.read_graph()
        ids, mds = ix.read_graph_metadata()
        assert_edge_rules(g, ids, mds, pop["md_bits"], pop["md_mags"], levels, nb, nb0)
        slot_scores_exact(ix, pop["md_bits"], pop["md_mags"], levels, metric, st)
        codes, mags = ix.read_codes(0, n + 2)
        fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n, levels, nb, nb0, g["entry"], g["node_row"], g["adj"], g["child"])
        mg = pymeta.MdGraph(fg, pop["md_bits"], pop["md_mags"], ids, mds, 1)
        r_ids, r_scores, r_counts, r_err = ix.batch_search_filtered(q, filters, k, ef_search=64, shortlist_size=64)
        w = pymeta.search_batch_md(mg, raw, q, filters, k, ef_search=64)
        assert np.array_equal(r_err, w[3]) and np.array_equal(r_counts, w[2])
        assert np.array_equal(r_ids, w[0]) and np.array_equal(bits(r_scores), bits(w[1]))
        got_rows = {id_row.get(int(x), -1) for i in range(nq) for x in r_ids[i, : r_counts[i]]}
        assert not got_rows & deleted
        if frac == 0.1:   # recall against a fresh replica build over the live embeddings
            live = np.array([r == EMPTY or int(r) not in deleted for r in pop["row"]])
            fresh_pop = {c: pop[c][live] for c in ("row", "node_id", "base_id", "md_row", "max_level")}
            fresh_pop.update(md_bits=pop["md_bits"], md_mags=pop["md_mags"], main_root_md=pop["main_root_md"],
                             pseudo_root_md=pop["pseudo_root_md"])
            fx, ff = gpu_index(fresh_pop, vecs, st, metric, levels, nb, nb0, efc, 256)
            f_ids, _, f_counts, _ = fx.batch_search_filtered(q, filters, k, ef_search=64, shortlist_size=64)
            fx.close()
            for part in (0, 1):   # unfiltered, filtered
                sel = np.array([(f is not None) == bool(part) for f in filters])
                r_now = live_recall(vecs, pop, deleted, q[sel], [f for f, s_ in zip(filters, sel) if s_], r_ids[sel], r_counts[sel], k, id_row)
                r_fresh = live_recall(vecs, pop, deleted, q[sel], [f for f, s_ in zip(filters, sel) if s_], f_ids[sel], f_counts[sel], k,
                                      id_row)
                assert r_now >= r_fresh - 0.05, (part, r_now, r_fresh)
    ix.close()


def test_deleted_embeddings_never_come_back():
    levels, nb, nb0, efc, k = 4, 16, 32, 64, 20
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 48
    n = 3000
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=41)
    vecs = pop["vecs"]
    id_row = {int(i): int(r) for i, r in zip(pop["node_id"], pop["row"]) if r != EMPTY}
    ix, _ = gpu_index(pop, vecs, st, metric, levels, nb, nb0, efc, 256)
    rng = np.random.default_rng(9)
    victims = [int(r) for r in pick(pop, n, rng, 60)]
    ix.delete_rows_replicas(victims[:30], max_batch=1)
    ix.delete_rows_replicas(victims[30:])
    dead = set(victims)
    q, filters = [], []
    for r in victims:   # unfiltered, and filtered by each pattern its Metadata replicas carry
        q.append(vecs[r])
        filters.append(None)
        for m in pop["md_row"][(pop["row"] == r) & (pop["md_row"] != EMPTY)]:
            if pop["md_mags"][m] != 0:
                q.append(vecs[r])
                filters.append([pop["md_bits"][m].astype(np.int8)])
    q = np.array(q, np.float32)
    assert sum(f is not None for f in filters) >= 40
    r_ids, _, r_counts, _ = ix.batch_search_filtered(q, filters, k, ef_search=128, shortlist_size=64)
    got = {id_row.get(int(x), -1) for i in range(len(q)) for x in r_ids[i, : r_counts[i]]}
    assert got and not got & dead
    q = vecs[victims]
    for mode in (cdb.SearchMode.BRUTE_RAW, cdb.SearchMode.BRUTE_CODES, cdb.SearchMode.HNSW):
        ids_, _, counts, _ = ix.batch_search(q, k, mode, ef_search=128, shortlist_size=64)
        got = {int(x) for i in range(len(victims)) for x in ids_[i, : counts[i]]}
        if mode == cdb.SearchMode.HNSW:
            got = {id_row.get(x, -1) for x in got}
        assert got and not got & dead, mode
    ix.close()


def snapshot(ix):
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    sc = ix.read_replica_slot_scores()
    return len(ix), g, ids, mds, [bits(a) for a in sc], ix.deleted_rows()


def assert_same(s0, s1):
    assert s0[0] == s1[0]
    g0, g1 = s0[1], s1[1]
    assert all(g0[key] == g1[key] for key in ("num_levels", "neighbors_count", "level0_neighbors_count", "entry", "root_row"))
    for lv in range(g0["num_levels"] + 1):
        for key in ("node_row", "adj", "child"):
            assert np.array_equal(g0[key][lv], g1[key][lv]), (key, lv)
        for i in (2, 3, 4):
            assert np.array_equal(s0[i][lv], s1[i][lv]), (i, lv)
    assert np.array_equal(s0[5], s1[5])


def raw_delete(ix, rows, shortlist=64):
    import ctypes as C
    r = np.ascontiguousarray(rows, np.uint32)
    st = np.zeros(max(r.size, 1), np.uint8)
    done = C.c_uint64(7)
    rc = ix._lib.cdb_index_delete_rows_replicas(ix._h, r.ctypes.data, r.size, shortlist, 0, st.ctypes.data, C.byref(done))
    return rc, done.value


def test_refusals_leave_the_index_unchanged():
    levels, nb, nb0, efc = 3, 8, 16, 16
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 24
    n = 300
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=43)
    INV, UNS = int(cdb.Status.INVALID_PARAMS), int(cdb.Status.UNSUPPORTED)
    # no graph, and a graph without metadata: CDB_INVALID_PARAMS
    plain = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    plain.append(pop["vecs"])
    assert raw_delete(plain, [3]) == (INV, 0)
    plain.build_graph(levels, nb, nb0, efc, 64, 64, 1)
    g0 = plain.read_graph()
    assert raw_delete(plain, [3]) == (INV, 0)
    assert "cdb_index_delete_rows" in cdb._lib.load().cdb_last_error_string().decode()
    with pytest.raises(cdb.CosdataError) as e:
        plain.read_replica_slot_scores()
    assert e.value.status == cdb.Status.INVALID_PARAMS
    assert np.array_equal(plain.read_graph()["adj"][0], g0["adj"][0]) and not plain.deleted_rows().any()
    plain.close()
    ix, _ = gpu_index(pop, pop["vecs"], st, metric, levels, nb, nb0, efc, 64)
    assert ix.delete_rows_replicas([5, 6]).tolist() == [0, 0]
    s0 = snapshot(ix)
    for rows, sl, why in (([1, n + 2], 64, "out of range"), ([1, n], 64, "root rows"), ([n + 1], 64, "root rows"),
                          ([1], 0, "shortlist_size"), ([1], 65, "shortlist_size")):
        rc, done = raw_delete(ix, rows, sl)
        assert rc == INV and done in (0, 7), why                       # a shortlist_size refusal leaves *out_deleted alone
        assert why in cdb._lib.load().cdb_last_error_string().decode(), why
        assert_same(s0, snapshot(ix))
    assert raw_delete(ix, []) == (0, 0)
    assert_same(s0, snapshot(ix))
    # uploaded metadata: CDB_UNSUPPORTED for the delete and the slot scores
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    ix.set_graph_metadata(pop["md_bits"], pop["md_mags"], ids, mds, 1)
    marks = ix.deleted_rows()
    assert raw_delete(ix, [1]) == (UNS, 0)
    with pytest.raises(cdb.CosdataError) as e:
        ix.read_replica_slot_scores()
    assert e.value.status == cdb.Status.UNSUPPORTED
    g1 = ix.read_graph()
    assert all(np.array_equal(g["adj"][lv], g1["adj"][lv]) for lv in range(levels + 1))
    assert np.array_equal(marks, ix.deleted_rows())
    ix.close()


def test_a_search_enqueued_before_a_delete_sees_the_old_graph():
    import threading
    import torch
    levels, nb, nb0, efc, k, nq = 5, 16, 32, 64, 10, 256
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 48
    n = 5000
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=47)
    vecs = pop["vecs"]
    ix, _ = gpu_index(pop, vecs, st, metric, levels, nb, nb0, efc, 256)
    old_g = ix.read_graph()
    old_ids, old_mds = ix.read_graph_metadata()
    rng = np.random.default_rng(6)
    victims = rng.choice(n, n // 5, replace=False)
    queries = (vecs[victims[:nq]] + 0.01 * rng.normal(size=(nq, dim))).astype(np.float32).clip(-0.999, 0.999)
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
    s = ix.delete_rows_replicas(victims)
    deleted.set()
    t.join()
    assert not errors and (s != 1).all()
    for s_ in streams:
        s_.synchronize()
    new_g = ix.read_graph()
    new_ids, new_mds = ix.read_graph_metadata()
    codes, mags = ix.read_codes(0, n + 2)
    raw = np.concatenate([vecs, np.zeros((2, dim), np.float32)])
    for (g, ids_, mds_), (r_ids, r_sc, r_cnt) in zip(((old_g, old_ids, old_mds), (new_g, new_ids, new_mds)), out):
        fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n, levels, nb, nb0, g["entry"], g["node_row"], g["adj"], g["child"])
        mg = pymeta.MdGraph(fg, pop["md_bits"], pop["md_mags"], ids_, mds_, 1)
        w = pymeta.search_batch_md(mg, raw, queries, [None] * nq, k, ef_search=64)
        assert np.array_equal(r_ids.cpu().numpy().view(np.uint32), w[0])
        assert np.array_equal(bits(r_sc.cpu().numpy()), bits(w[1])) and np.array_equal(r_cnt.cpu().numpy().view(np.uint32), w[2])
    # only the first search returns the deleted embeddings
    dead_ids = set(pop["node_id"][np.isin(pop["row"], victims)].tolist())
    got = [set(x.cpu().numpy().view(np.uint32).ravel().tolist()) for x in (out[0][0], out[1][0])]
    assert (got[0] & dead_ids) and not (got[1] & dead_ids)
    ix.close()
