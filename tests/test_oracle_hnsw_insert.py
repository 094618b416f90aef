"""The insert oracle (tests/hnsw_insert_oracle.c) against the pinned builder: a build is the root plus an insert of every
row, a graph loaded from storage gets the reference's reload state, and recomputed slot similarities equal the stored
ones (every plain arm is symmetric)."""
import numpy as np
import pytest

import oracle as orc
from oracle import pyhnsw
from tests import pyinsert

ST_F16, ST_U8, ST_SUB2 = 4, 0, 2
COS, DOT = 0, 3
EMPTY = 0xFFFFFFFF


def clustered(n, dim, seed):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(8, dim)).astype(np.float32)
    v = (centres[rng.integers(0, 8, n)] + 0.35 * rng.normal(size=(n, dim))).astype(np.float32)
    return (v / (np.abs(v).max() * 1.01)).astype(np.float32)


def table(st, vecs, root):
    return orc.quantize_batch(st, np.concatenate([vecs, root[None]]).astype(np.float32))


@pytest.mark.parametrize("st,metric,chunk", [(ST_F16, COS, 1), (ST_F16, COS, 7), (ST_F16, COS, None), (ST_U8, COS, 7),
                                             (ST_SUB2, DOT, 7), (ST_F16, DOT, None)])
def test_build_is_init_plus_insert(st, metric, chunk):
    n, dim, levels, nb, nb0, efc, seed = 400, 16, 3, 8, 16, 24, 3
    vecs = clustered(n, dim, 1)
    root = np.linspace(-0.9, 0.9, dim).astype(np.float32)
    fg = pyhnsw.build(metric, st, vecs, root, num_levels=levels, neighbors_count=nb, level0_neighbors_count=nb0,
                      ef_construction=efc, seed=seed)
    codes, mags = table(st, vecs, root)
    g = pyinsert.Graph.init(metric, st, dim, codes, mags, n, levels, nb, nb0)
    step = chunk or n
    for first in range(0, n, step):
        assert g.insert(first, min(step, n - first), ef_construction=efc, seed=seed).sum() == 0
    e = g.export()
    assert e["entry"] == fg.entry
    for lv in range(levels + 1):
        assert np.array_equal(e["node_row"][lv], fg.node_row[lv]), lv
        assert np.array_equal(e["adj"][lv], fg.adj[lv]), lv
        if lv:
            assert np.array_equal(e["child"][lv], fg.child[lv]), lv
    g.close()


@pytest.mark.parametrize("st,metric", [(ST_F16, COS), (ST_U8, COS), (ST_SUB2, DOT), (ST_F16, DOT)])
def test_reload_recomputes_the_stored_similarities(st, metric):
    n, dim, levels, nb, nb0 = 300, 24, 2, 6, 8
    vecs = clustered(n, dim, 7)
    root = np.linspace(-0.5, 0.5, dim).astype(np.float32)
    codes, mags = table(st, vecs, root)
    g = pyinsert.Graph.init(metric, st, dim, codes, mags, n, levels, nb, nb0)
    g.insert(0, n, ef_construction=16)
    built = g.export()
    r = pyinsert.Graph.from_graph(metric, st, dim, codes, mags, built)
    re = r.export()
    for lv in range(levels + 1):
        filled = built["adj"][lv] != EMPTY
        assert filled.sum() > 0
        assert np.array_equal(re["simkey"][lv][filled], built["simkey"][lv][filled]), lv
    g.close()
    r.close()


def test_reload_lowest_index_matches_prob_node_rule():
    # duplicated rows give tied similarities; a tiny level-0 degree gives full nodes; upper levels keep empty slots
    n, dim, levels, nb, nb0 = 240, 12, 2, 8, 4
    base = clustered(n // 3, dim, 9)
    vecs = np.concatenate([base, base, base]).astype(np.float32)
    root = np.linspace(-0.3, 0.3, dim).astype(np.float32)
    codes, mags = table(ST_U8, vecs, root)
    g = pyinsert.Graph.init(COS, ST_U8, dim, codes, mags, n, levels, nb, nb0)
    g.insert(0, n, ef_construction=16)
    built = g.export()
    r = pyinsert.Graph.from_graph(COS, ST_U8, dim, codes, mags, built)
    re = r.export()
    mn, mx = pyinsert.min_max_keys(COS)
    saw_full = saw_empty = saw_tie = False
    for lv in range(levels + 1):
        nbc = nb0 if lv == 0 else nb
        li, lk = pyinsert.reload_lowest(re["simkey"][lv], re["adj"][lv], nbc, mn, mx)
        assert np.array_equal(li, re["lowest_idx"][lv]) and np.array_equal(lk, re["lowest_key"][lv]), lv
        adj = re["adj"][lv].reshape(-1, nbc)
        keys = re["simkey"][lv].reshape(-1, nbc)
        full = (adj != EMPTY).all(1)
        saw_full |= bool(full.any())
        saw_empty |= bool((~full).any())
        saw_tie |= any(len(set(k.tolist())) < nbc for k in keys[full])
    assert saw_full and saw_empty and saw_tie
    g.close()
    r.close()


def test_insert_after_build_searches_a_mid_table_root():
    n0, n1, dim = 300, 120, 16
    vecs = clustered(n0 + n1, dim, 5)
    root = np.linspace(-0.7, 0.7, dim).astype(np.float32)
    allv = np.concatenate([vecs[:n0], root[None], vecs[n0:]]).astype(np.float32)
    codes, mags = orc.quantize_batch(ST_F16, allv)
    g = pyinsert.Graph.init(COS, ST_F16, dim, codes, mags, n0, 3, 8, 16)
    g.insert(0, n0, ef_construction=24)
    assert g.insert(n0 + 1, n1, ef_construction=24).sum() == 0
    e = g.export()
    assert e["node_row"][0].size == n0 + n1 + 1 and e["node_row"][1][0] == n0
    deg = (e["adj"][0].reshape(-1, 16) != EMPTY).sum(1)
    assert (deg[n0 + 1:] > 0).all()
    ids, scores, counts, err, ev, pops = g.search_batch(allv, allv[n0 + 1:n0 + 41], 5, ef_search=32)
    assert (err == 0).all() and not (ids == n0).any()
    assert np.mean(ids[:, 0] == np.arange(n0 + 1, n0 + 41)) > 0.9
    g.close()


def test_insert_graph_argument_checks():
    from cosdata_b200.api import check_insert_args
    assert check_insert_args(128, 64, 4096) is None
    assert check_insert_args(1, 1, 0, [0, 3, 9], 3).dtype == np.uint8
    for bad in [(0, 64, 1), (4097, 64, 1), (128, 0, 1), (128, 65, 1), (128, 64, -1)]:
        with pytest.raises(ValueError):
            check_insert_args(*bad)
    with pytest.raises(ValueError, match="one draw per new row"):
        check_insert_args(128, 64, 1, [1, 2], 3)
    with pytest.raises(ValueError, match="u8"):
        check_insert_args(128, 64, 1, [1, 256], 2)
