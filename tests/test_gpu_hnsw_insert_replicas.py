"""cdb_index_insert_graph_replicas: more nodes of a collection with a metadata schema go into the replica graph on the GPU.
  * one node at a time, a build of A followed by inserts of B equals the oracle's replica build of A+B array for array
    (the reference builds by repeated insertion, so the pinned oracle is the target), failed flags included;
  * batched inserts keep the replica edge rules, CUDA search (filtered and unfiltered) equals the oracle's on the grown graph,
    filtered queries only return replicas carrying the filter's pattern, and recall stays near a one-shot build;
  * refusals leave the index unchanged, and a search enqueued before an insert sees the old graph."""
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from oracle import pymeta

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
EMPTY = 0xFFFFFFFF
PSEUDO_ROOT_ID = 0xFFFFFFFF - 257


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def grown_population(n, n_a, dim, levels, n_patterns=7, seed=13, zero=False, b_only=2, chunks=3, pseudo_in_b=False):
    """replica_population(n) split into A (pseudo replicas + embeddings < n_a) and B (the rest).  The last `b_only` patterns
    are carried only by B's embeddings (their pseudo replicas exist from the start, as the reference creates them with the
    collection).  B's metadata replicas partly name new Metadata table rows (copies of those patterns) appended through
    md_bits_new: new_rows[c] = the rows the c-th of `chunks` insert calls appends.  Rows of B are index rows: embeddings
    >= n_a sit behind the two roots the build appends.  zero: the first B embedding with metadata replicas gets a zero
    vector.  pseudo_in_b: B starts with one more pseudo replica (its traversal meets metadata replicas, the reference's
    unreachable!() arm: the insert fails)."""
    from tests import mdgraph
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, n_patterns=n_patterns, seed=seed)
    rng = np.random.default_rng(seed + 100)
    vecs = pop["vecs"].copy()
    cols = ("row", "node_id", "base_id", "md_row", "max_level")
    is_b = (pop["row"] != EMPTY) & (pop["row"] >= n_a)
    first_b_only = 2 + n_patterns - b_only
    a = {c: pop[c][~is_b].copy() for c in cols}
    a["md_row"][(a["row"] != EMPTY) & (a["md_row"] >= first_b_only)] -= b_only
    b = {c: list(pop[c][is_b]) for c in cols}
    b["row"] = [r + 2 for r in b["row"]]
    if zero:
        e = next(int(r) - 2 for r, m in zip(b["row"], b["md_row"]) if m >= 2)
        vecs[e] = 0.0
    if pseudo_in_b:
        for c, v in zip(cols, (EMPTY, PSEUDO_ROOT_ID + 1 + n_patterns, PSEUDO_ROOT_ID, 2, 1)):
            b[c].insert(0, v)
    b = {c: np.array(b[c], np.uint8 if c == "max_level" else np.uint32) for c in cols}
    n_md0 = pop["md_bits"].shape[0]
    new_bits = pop["md_bits"][first_b_only:first_b_only + b_only].copy()
    new_mags = pop["md_mags"][first_b_only:first_b_only + b_only].copy()
    nb = b["row"].size
    bounds = [nb * c // chunks for c in range(chunks + 1)]
    new_rows = [[] for _ in range(chunks)]
    for p in range(b_only):
        new_rows[min(p, chunks - 1)].append(p)
    call_of = np.searchsorted(bounds, np.arange(nb), side="right") - 1
    for t in range(nb):   # half the replicas of a B-only pattern name its new table row, once the call appending it has come
        p = int(b["md_row"][t]) - first_b_only
        if b["row"][t] != EMPTY and 0 <= p < b_only and min(p, chunks - 1) <= call_of[t] and rng.random() < 0.5:
            b["md_row"][t] = n_md0 + p
    return dict(vecs=vecs, a=a, b=b, bounds=bounds, new_rows=new_rows, md_bits=pop["md_bits"], md_mags=pop["md_mags"],
                new_bits=new_bits, new_mags=new_mags, n=n, n_a=n_a, main_root_md=pop["main_root_md"],
                pseudo_root_md=pop["pseudo_root_md"], b_only_patterns=new_bits)


def build_a(gp, st, metric, levels, nb, nb0, efc, max_batch, extra_cap=0):
    n, n_a = gp["n"], gp["n_a"]
    dim = gp["vecs"].shape[1]
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2 + extra_cap, keep_raw_f32=True)
    ix.append(gp["vecs"][:n_a])
    a = gp["a"]
    failed = ix.build_graph_replicas(a["row"], a["node_id"], a["base_id"], a["md_row"], a["max_level"], gp["md_bits"], gp["md_mags"],
                                     gp["main_root_md"], gp["pseudo_root_md"], levels, nb, nb0, efc, 64, max_batch, 1)
    ix.append(gp["vecs"][n_a:])
    return ix, failed


def insert_b(ix, gp, efc, max_batch, calls):
    """B in `calls` insert calls (1 or len(gp['new_rows'])) -> failed over B"""
    b, out = gp["b"], []
    spans = [(0, b["row"].size, list(range(gp["new_bits"].shape[0])))] if calls == 1 else \
        [(gp["bounds"][c], gp["bounds"][c + 1], gp["new_rows"][c]) for c in range(calls)]
    for lo, hi, rows in spans:
        out.append(ix.insert_graph_replicas(b["row"][lo:hi], b["node_id"][lo:hi], b["base_id"][lo:hi], b["md_row"][lo:hi],
                                            b["max_level"][lo:hi], gp["new_bits"][rows], gp["new_mags"][rows], efc, 64, max_batch))
        assert out[-1].size == hi - lo
    return np.concatenate(out)


def full_table(gp):
    return np.concatenate([gp["md_bits"], gp["new_bits"]]), np.concatenate([gp["md_mags"], gp["new_mags"]])


def oracle_grown(ix, gp, st, metric, levels, nb, nb0, efc):
    n, n_a = gp["n"], gp["n_a"]
    dim = gp["vecs"].shape[1]
    codes, mags = ix.read_codes(0, n + 2)
    a, b = gp["a"], gp["b"]
    cat = {c: np.concatenate([a[c], b[c]]) for c in a}
    rows = np.where(cat["row"] == EMPTY, n_a + 1, cat["row"]).astype(np.uint32)
    rl = pymeta.ReplicaList(rows, cat["node_id"], cat["base_id"], cat["md_row"], cat["max_level"], n_a, gp["main_root_md"], n_a + 1,
                            gp["pseudo_root_md"])
    md_bits, md_mags = full_table(gp)
    return pymeta.build_md(int(metric), int(st), dim, codes, mags, md_bits, md_mags, rl, num_levels=levels, neighbors_count=nb,
                           level0_neighbors_count=nb0, ef_construction=efc)


def without_nodes(node_row, node_id, node_md, adj, child, nbs, drop_ids):
    """the level arrays with every node whose id is in drop_ids removed; those nodes must be isolated (no slot of theirs
    filled, no slot naming them, no child pointer at them)"""
    out = dict(node_row=[], node_id=[], node_md=[], adj=[], child=[])
    remap = None
    for lv in range(len(node_row)):
        keep = ~np.isin(node_id[lv], drop_ids)
        a = adj[lv].reshape(-1, nbs[lv])
        assert (a[~keep] == EMPTY).all(), lv
        new_index = np.full(keep.size + 1, EMPTY, np.int64)
        new_index[np.flatnonzero(keep)] = np.arange(int(keep.sum()))
        ak = a[keep].astype(np.int64)
        ak = np.where(ak == EMPTY, keep.size, ak)
        mapped = new_index[ak]
        assert ((mapped != EMPTY) | (ak == keep.size)).all(), lv     # no link to a removed node
        out["adj"].append(np.where(ak == keep.size, EMPTY, mapped).astype(np.uint32).ravel())
        for key, arr in (("node_row", node_row), ("node_id", node_id), ("node_md", node_md)):
            out[key].append(arr[lv][keep])
        if lv:
            c = remap[child[lv][keep].astype(np.int64)]
            assert (c != EMPTY).all(), lv
            out["child"].append(c.astype(np.uint32))
        else:
            out["child"].append(None)
        remap = new_index
    return out


def assert_md_graph_equal(ix, mg, levels, failed_ids=()):
    """GPU graph == oracle graph array for array.  An entry whose insert failed keeps isolated nodes on every level it drew
    here, while the oracle (like the reference) keeps those created above the level whose traversal failed: both sides are
    compared without the failed entries' nodes, which must be isolated on both."""
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    assert g["entry"] == mg.fg.entry == 0 and mg.pseudo_entry == 1
    nbs = [g["level0_neighbors_count"]] + [g["neighbors_count"]] * levels
    drop = np.array(list(failed_ids), np.uint32)
    got = without_nodes(g["node_row"], ids, mds, g["adj"], g["child"], nbs, drop)
    want = without_nodes(mg.fg.node_row, mg.node_id, mg.node_md, mg.fg.adj, mg.fg.child, nbs, drop)
    for lv in range(levels + 1):
        for key in ("node_row", "node_id", "node_md", "adj") + (("child",) if lv else ()):
            assert np.array_equal(got[key][lv], want[key][lv]), (key, lv)
    if not drop.size:
        for lv in range(levels + 1):
            assert ids[lv].size == mg.node_id[lv].size, lv


@pytest.mark.parametrize("st,metric,dim,nb0", [(ST.HalfPrecisionFP, MK.Cosine, 32, 16), (ST.UnsignedByte, MK.Cosine, 32, 16),
                                               (ST.SubByte2, MK.DotProduct, 32, 16), (ST.FullPrecisionFP, MK.Cosine, 32, 16),
                                               (ST.HalfPrecisionFP, MK.Cosine, 768, 64)])
def test_sequential_insert_equals_oracle_replica_build(st, metric, dim, nb0):
    levels, nb, efc = 4, 8, 32
    n, n_a = (500, 300) if dim == 32 else (240, 150)
    gp = grown_population(n, n_a, dim, levels, seed=13, zero=True, pseudo_in_b=True)
    mg, ofailed = oracle_grown(build_a(gp, st, metric, levels, nb, nb0, efc, 1)[0], gp, st, metric, levels, nb, nb0, efc)
    n_a_nodes = gp["a"]["row"].size
    if metric == MK.Cosine and st in (ST.HalfPrecisionFP, ST.FullPrecisionFP):
        assert ofailed[n_a_nodes + 1:].any()                            # the zero-norm embedding's base replica fails
    if metric == MK.Cosine:                                             # only cosine has the replica arms
        assert ofailed[n_a_nodes] == 1                                  # the pseudo replica of B meets (Metadata, Pseudo)
    assert not ofailed[:n_a_nodes].any()
    all_ids = np.concatenate([gp["a"]["node_id"], gp["b"]["node_id"]])
    for calls in (1, 3):
        ix, fa = build_a(gp, st, metric, levels, nb, nb0, efc, 1)
        fb = insert_b(ix, gp, efc, 1, calls)
        assert np.array_equal(np.concatenate([fa, fb]), ofailed), calls
        assert_md_graph_equal(ix, mg, levels, all_ids[ofailed != 0])
        assert len(ix) == n + 2
        ix.close()


def assert_edge_rules(g, ids, mds, md_bits, md_mags, levels, nb, nb0):
    # the replica rules (vector_store.rs:1014-1040) hold on every edge
    for lv in range(levels + 1):
        nbc = nb0 if lv == 0 else nb
        adj = g["adj"][lv].reshape(-1, nbc)
        has = (mds[lv] != EMPTY) & (md_mags[np.minimum(mds[lv], md_mags.size - 1)] != 0)
        a_idx, slot = np.nonzero(adj != EMPTY)
        b_idx = adj[a_idx, slot]
        assert np.array_equal(has[a_idx], has[b_idx]), lv                           # Base nodes never meet the pseudo component
        both = has[a_idx]
        pa, pb = md_bits[mds[lv][a_idx[both]]], md_bits[mds[lv][b_idx[both]]]
        is_ps = lambda x: (ids[lv][x] >= 0xFFFFFFFF - 257) & (ids[lv][x] <= 0xFFFFFFFF - 2)
        mixed = ~(is_ps(a_idx[both]) & is_ps(b_idx[both]))                           # at least one Metadata end: identical dims
        assert np.array_equal(pa[mixed], pb[mixed]), lv
        if lv >= 1:
            assert np.array_equal(g["node_row"][lv - 1][g["child"][lv]], g["node_row"][lv])


def recall(r_ids, r_counts, gt, k):
    return np.mean([len(set((r_ids[i, : r_counts[i]] // 4).tolist()) & set(gt[i].tolist())) / k for i in range(len(gt))])


def test_batched_inserts_rules_search_parity_filters_and_recall():
    levels, nb, nb0, efc, k = 5, 16, 32, 64, 10
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 48
    n, n_a = 6000, 4000
    gp = grown_population(n, n_a, dim, levels, seed=17, chunks=10)
    vecs = gp["vecs"]
    md_bits, md_mags = full_table(gp)
    b_only = gp["b_only_patterns"]
    # queries: unfiltered, every pattern, and every third one a pattern only B's embeddings carry
    rng = np.random.default_rng(4)
    nq = 90
    q = (vecs[rng.integers(0, n, nq)] + 0.03 * rng.normal(size=(nq, dim))).astype(np.float32).clip(-0.999, 0.999)
    pats = gp["md_bits"][2:]
    filters = [None if i % 3 == 0 else [(b_only[(i // 3) % len(b_only)] if i % 3 == 1 else pats[i % len(pats)]).astype(np.int8)]
               for i in range(nq)]
    is_b_only = lambda f: (b_only == f.astype(np.int32)).all(1).any()
    # exact top-k over the embeddings that qualify (unfiltered: all; filtered: those with a replica of the pattern)
    b = gp["b"]
    all_rows = np.concatenate([gp["a"]["row"], np.where(b["row"] == EMPTY, EMPTY, b["row"] - 2).astype(np.uint32)])
    all_md = np.concatenate([gp["a"]["md_row"], b["md_row"]])
    all_id = np.concatenate([gp["a"]["node_id"], b["node_id"]])
    id_to_md = dict(zip(all_id.tolist(), all_md.tolist()))
    gt = np.zeros((nq, k), np.int64)
    for i in range(nq):
        if filters[i] is None:
            cand = np.arange(n)
        else:
            carries = (all_md != EMPTY) & (md_bits[np.minimum(all_md, md_bits.shape[0] - 1)] == filters[i][0]).all(1)
            cand = np.unique(all_rows[carries & (all_rows != EMPTY)])
        ids_, _ = orc.brute_topk_f32(vecs[cand], q[i:i + 1], min(k, cand.size))
        gt[i, : ids_.shape[1]] = cand[ids_[0]]
    # the one-shot batched build over the same nodes (rows in vecs order, roots behind them)
    one = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2, keep_raw_f32=True)
    one.append(vecs)
    f1 = one.build_graph_replicas(all_rows, all_id, np.concatenate([gp["a"]["base_id"], b["base_id"]]), all_md,
                                  np.concatenate([gp["a"]["max_level"], b["max_level"]]), md_bits, md_mags, gp["main_root_md"],
                                  gp["pseudo_root_md"], levels, nb, nb0, efc, 64, 256, 1)
    assert f1.sum() == 0
    i1, _, c1, _ = one.batch_search_filtered(q, filters, k, ef_search=64, shortlist_size=64)
    one.close()
    r1 = recall(i1, c1, gt, k)
    for calls in (1, 10):
        ix, fa = build_a(gp, st, metric, levels, nb, nb0, efc, 256)
        fb = insert_b(ix, gp, efc, 256, calls)
        assert fa.sum() == 0 and fb.sum() == 0
        g = ix.read_graph()
        ids, mds = ix.read_graph_metadata()
        assert all(np.array_equal(ids[lv][:2], [EMPTY, PSEUDO_ROOT_ID]) for lv in range(levels + 1))
        assert ids[0].size == 2 + all_id.size and np.array_equal(ids[0][2:], all_id)
        assert_edge_rules(g, ids, mds, md_bits, md_mags, levels, nb, nb0)
        deg0 = (g["adj"][0].reshape(-1, nb0) != EMPTY).sum(1)
        assert (deg0[2 + gp["a"]["row"].size:] > 0).mean() > 0.99
        # CUDA search == oracle search on the exported graph: ids, score bits, counts and error flags
        codes, mags = ix.read_codes(0, n + 2)
        from oracle import pyhnsw
        fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n_a, levels, nb, nb0, g["entry"], g["node_row"], g["adj"], g["child"])
        mg = pymeta.MdGraph(fg, md_bits, md_mags, ids, mds, 1)
        raw = np.concatenate([vecs[:n_a], np.zeros((2, dim), np.float32), vecs[n_a:]])
        r_ids, r_scores, r_counts, r_err = ix.batch_search_filtered(q, filters, k, ef_search=64, shortlist_size=64)
        w = pymeta.search_batch_md(mg, raw, q, filters, k, ef_search=64)
        assert np.array_equal(r_err, w[3]) and np.array_equal(r_counts, w[2])
        assert np.array_equal(r_ids, w[0]) and np.array_equal(bits(r_scores), bits(w[1]))
        # a filtered query only returns replicas that carry its pattern, the B-only patterns included
        new_hits = 0
        for i in range(nq):
            got = r_ids[i, : r_counts[i]]
            if filters[i] is None:
                assert all(id_to_md[int(x)] == 0 for x in got) and r_counts[i] == k
                continue
            assert all((md_bits[id_to_md[int(x)]] == filters[i][0]).all() for x in got), i
            new_hits += int(r_counts[i]) if is_b_only(filters[i][0]) else 0
        assert new_hits > 0.5 * k * sum(f is not None and is_b_only(f[0]) for f in filters)
        r = recall(r_ids, r_counts, gt, k)
        assert r >= r1 - 0.05, (calls, r, r1)
        ix.close()


def snapshot(ix):
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    return len(ix), g, ids, mds


def assert_same(s0, s1):
    assert s0[0] == s1[0]
    g0, g1 = s0[1], s1[1]
    assert all(g0[key] == g1[key] for key in ("num_levels", "neighbors_count", "level0_neighbors_count", "entry", "root_row"))
    for lv in range(g0["num_levels"] + 1):
        for key in ("node_row", "adj", "child"):
            assert np.array_equal(g0[key][lv], g1[key][lv]), (key, lv)
        assert np.array_equal(s0[2][lv], s1[2][lv]) and np.array_equal(s0[3][lv], s1[3][lv]), lv


def raw_insert(ix, b, lo, hi, md_dims=6, num_levels=3, nb=8, nb0=16, efc=16, max_level=True, new_bits=None, new_mags=None):
    from cosdata_b200._lib import BuildParams, ReplicaInsert
    arrs = [np.ascontiguousarray(b[c][lo:hi], np.uint32) for c in ("row", "node_id", "base_id", "md_row")]
    lv = np.ascontiguousarray(b["max_level"][lo:hi], np.uint8)
    nbits = np.zeros((0, md_dims), np.int32) if new_bits is None else np.ascontiguousarray(new_bits, np.int32)
    nmags = np.zeros(0, np.float32) if new_mags is None else np.ascontiguousarray(new_mags, np.float32)
    ri = ReplicaInsert(hi - lo, *[a.ctypes.data for a in arrs], lv.ctypes.data if max_level else None, md_dims, nbits.shape[0],
                       nbits.ctypes.data, nmags.ctypes.data)
    bp = BuildParams(num_levels, nb, nb0, efc, 64, 64, 0)
    done = C.c_uint64(7)
    rc = ix._lib.cdb_index_insert_graph_replicas(ix._h, C.byref(bp), C.byref(ri), None, C.byref(done))
    return rc, done.value


def test_refusals_leave_the_index_unchanged():
    levels, nb, nb0, efc = 3, 8, 16, 16
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 24
    gp = grown_population(300, 200, dim, levels, seed=5)
    b = gp["b"]
    nbn = b["row"].size
    INV, UNS = int(cdb.Status.INVALID_PARAMS), int(cdb.Status.UNSUPPORTED)
    # no graph, and a graph without metadata: CDB_INVALID_PARAMS
    plain = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=400, keep_raw_f32=True)
    plain.append(gp["vecs"])
    assert raw_insert(plain, b, 0, 4)[0] == INV
    plain.build_graph(levels, nb, nb0, efc, 64, 64, 1)
    g0 = plain.read_graph()
    assert raw_insert(plain, b, 0, 4) == (INV, 0)
    assert "cdb_index_insert_graph" in cdb._lib.load().cdb_last_error_string().decode()
    assert np.array_equal(plain.read_graph()["adj"][0], g0["adj"][0])
    plain.close()
    ix, _ = build_a(gp, st, metric, levels, nb, nb0, efc, 64)
    s0 = snapshot(ix)
    n, n_a, n_md0 = gp["n"], gp["n_a"], gp["md_bits"].shape[0]
    md_full = n_md0 + gp["new_bits"].shape[0]
    ok = {c: b[c][:6].copy() for c in b}
    ok["md_row"][ok["md_row"] >= n_md0] = 2                            # only rows of the existing table

    def bad(key=None, t=0, v=0):
        bb = {c: ok[c].copy() for c in ok}
        if key:
            bb[key][t] = v
        return bb
    new_rows = dict(new_bits=gp["new_bits"], new_mags=gp["new_mags"])
    cases = [
        (bad("row", 2, n + 2), {}, "row out of range"),
        (bad("row", 2, n_a), {}, "root rows"),                        # the main root's row
        (bad("row", 3, n_a + 1), {}, "root rows"),                    # the pseudo root's row
        (bad("md_row", 1, n_md0), {}, "md_row out of range"),         # a table row the call does not append
        (bad("md_row", 1, md_full), new_rows, "md_row out of range"),
        (bad(), dict(md_dims=5), "md_dims"),
        (bad(), dict(num_levels=levels + 1), "differ from the graph"),
        (bad(), dict(nb0=nb0 * 2), "differ from the graph"),
        (bad(), dict(max_level=False), "null replica list"),
    ]
    for bb, kw, why in cases:
        args = dict(num_levels=levels, nb=nb, nb0=nb0, efc=efc)
        args.update(kw)
        assert raw_insert(ix, bb, 0, 6, **args) == (INV, 0), why
        assert why in cdb._lib.load().cdb_last_error_string().decode(), why
        assert_same(s0, snapshot(ix))
    # n_nodes == 0: CDB_OK, nothing inserted
    assert raw_insert(ix, b, 0, 0, num_levels=levels, nb=nb, nb0=nb0, efc=efc) == (0, 0)
    assert_same(s0, snapshot(ix))
    # grow it once; the plain writers stay unsupported on the grown graph
    failed = ix.insert_graph_replicas(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], gp["new_bits"], gp["new_mags"],
                                      efc, 64, 64)
    assert failed.size == nbn and failed.sum() == 0
    s1 = snapshot(ix)
    assert s1[2][0].size == s0[2][0].size + nbn
    with pytest.raises(cdb.CosdataError) as e:
        ix.insert_graph(efc, 64, 64, 1)
    assert e.value.status == cdb.Status.UNSUPPORTED
    with pytest.raises(cdb.CosdataError) as e:
        ix.delete_rows([0])
    assert e.value.status == cdb.Status.UNSUPPORTED
    with pytest.raises(cdb.CosdataError) as e:
        ix.read_graph_slot_scores()
    assert e.value.status == cdb.Status.UNSUPPORTED
    assert_same(s1, snapshot(ix))
    # uploaded metadata (over the replica build's own graph): CDB_UNSUPPORTED
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    md_bits, md_mags = full_table(gp)
    ix.set_graph_metadata(md_bits, md_mags, ids, mds, 1)
    assert raw_insert(ix, b, 0, 4, num_levels=levels, nb=nb, nb0=nb0, efc=efc) == (UNS, 0)
    assert_same(s1, snapshot(ix))
    up = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2, keep_raw_f32=True)
    up.append(np.concatenate([gp["vecs"][:n_a], np.zeros((2, dim), np.float32), gp["vecs"][n_a:]]))
    up.set_graph(g["num_levels"], nb, nb0, g["entry"], g["root_row"], g["node_row"], g["adj"], g["child"])
    up.set_graph_metadata(md_bits, md_mags, ids, mds, 1)
    su = snapshot(up)
    assert raw_insert(up, b, 0, 4, num_levels=levels, nb=nb, nb0=nb0, efc=efc) == (UNS, 0)
    assert_same(su, snapshot(up))
    up.close()
    ix.close()


def test_deleted_row_is_refused():
    levels, nb, nb0, efc = 3, 8, 16, 16
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 24
    gp = grown_population(300, 200, dim, levels, seed=5)
    n, n_a = gp["n"], gp["n_a"]
    b = gp["b"]
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2, keep_raw_f32=True)
    ix.append(gp["vecs"][:n_a])
    victim = int(gp["a"]["row"][-1])                                   # an A embedding, deleted before the build
    assert ix.delete_rows([victim]).tolist() == [0]
    a = {c: gp["a"][c][gp["a"]["row"] != victim] for c in gp["a"]}
    ix.build_graph_replicas(a["row"], a["node_id"], a["base_id"], a["md_row"], a["max_level"], gp["md_bits"], gp["md_mags"],
                            gp["main_root_md"], gp["pseudo_root_md"], levels, nb, nb0, efc, 64, 64, 1)
    ix.append(gp["vecs"][n_a:])
    s0 = snapshot(ix)
    bb = {c: b[c][:5].copy() for c in b}
    bb["row"][2] = victim
    assert raw_insert(ix, bb, 0, 5, num_levels=levels, nb=nb, nb0=nb0, efc=efc) == (int(cdb.Status.INVALID_PARAMS), 0)
    assert "deleted" in cdb._lib.load().cdb_last_error_string().decode()
    assert_same(s0, snapshot(ix))
    ix.close()


def test_shared_memory_check_refuses_before_any_change():
    # f32 x 12288 at ef_construction 4096 needs more shared memory per block than an H100 allows (hnsw_build_smem_check)
    levels, nb, nb0 = 2, 8, 16
    dim = 12288
    gp = grown_population(40, 30, dim, levels, seed=9)
    ix, _ = build_a(gp, ST.FullPrecisionFP, MK.Cosine, levels, nb, nb0, 16, 64)
    s0 = snapshot(ix)
    b = gp["b"]
    rc, done = raw_insert(ix, b, 0, b["row"].size, num_levels=levels, nb=nb, nb0=nb0, efc=4096,
                          new_bits=gp["new_bits"], new_mags=gp["new_mags"])
    assert (rc, done) == (int(cdb.Status.INVALID_PARAMS), 0)
    assert "shared memory" in cdb._lib.load().cdb_last_error_string().decode()
    assert_same(s0, snapshot(ix))
    failed = ix.insert_graph_replicas(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], gp["new_bits"], gp["new_mags"],
                                      16, 64, 64)
    assert failed.size == b["row"].size
    ix.close()


def test_a_search_enqueued_before_an_insert_sees_the_old_graph():
    import threading
    import torch
    levels, nb, nb0, efc, k, nq = 5, 16, 32, 64, 10, 256
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 48
    n, n_a = 5000, 4000
    gp = grown_population(n, n_a, dim, levels, seed=31)
    vecs = gp["vecs"]
    ix, _ = build_a(gp, st, metric, levels, nb, nb0, efc, 256)
    old_g = ix.read_graph()
    old_ids, old_mds = ix.read_graph_metadata()
    rng = np.random.default_rng(6)
    queries = (vecs[rng.integers(n_a, n, nq)] + 0.03 * rng.normal(size=(nq, dim))).astype(np.float32).clip(-0.999, 0.999)
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
    b = gp["b"]
    failed = ix.insert_graph_replicas(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], gp["new_bits"], gp["new_mags"],
                                      efc, 64, 256)
    inserted.set()
    t.join()
    assert not errors and failed.size == b["row"].size and failed.sum() == 0
    for s_ in streams:
        s_.synchronize()
    new_g = ix.read_graph()
    new_ids, new_mds = ix.read_graph_metadata()
    codes, mags = ix.read_codes(0, n + 2)
    raw = np.concatenate([vecs[:n_a], np.zeros((2, dim), np.float32), vecs[n_a:]])
    from oracle import pyhnsw
    old_bits, old_mags = gp["md_bits"], gp["md_mags"]
    md_bits, md_mags = full_table(gp)
    for (g, ids_, mds_, tb, tm), (r_ids, r_sc, r_cnt) in zip(((old_g, old_ids, old_mds, old_bits, old_mags),
                                                               (new_g, new_ids, new_mds, md_bits, md_mags)), out):
        fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n_a, levels, nb, nb0, g["entry"], g["node_row"], g["adj"], g["child"])
        mg = pymeta.MdGraph(fg, tb, tm, ids_, mds_, 1)
        w = pymeta.search_batch_md(mg, raw, queries, [None] * nq, k, ef_search=64)
        assert np.array_equal(r_ids.cpu().numpy().view(np.uint32), w[0])
        assert np.array_equal(bits(r_sc.cpu().numpy()), bits(w[1])) and np.array_equal(r_cnt.cpu().numpy().view(np.uint32), w[2])
    # only the second search reaches the new embeddings' replicas
    new_ids_set = set(b["node_id"].tolist())
    got = [set(x.cpu().numpy().view(np.uint32).ravel().tolist()) for x in (out[0][0], out[1][0])]
    assert not (got[0] & new_ids_set) and (got[1] & new_ids_set)
    ix.close()
