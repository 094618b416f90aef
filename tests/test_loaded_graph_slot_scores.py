"""Graphs loaded from the reference's index files with their stored slot similarities (CPU tests):
  * cdb_hnsw_files_slot_scores returns every written MetricResult (value and tag) bit for bit in adjacency order, 0 / 0xFF on
    empty slots, and damaged files still fail;
  * the oracle's reload (tests/hnsw_loaded_md_oracle.c) gives back the arrays and slot values of a build, and its
    lowest_index is prob_node.rs:155-169 restated in Python, ties, all-full nodes and MetricResult::max included;
  * reloaded without a pseudo root (a collection without a metadata schema), its inserts and deletes equal the plain insert
    and delete oracles on the same graph."""
import os

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from tests import mdgraph, pydelete_md
from tests.scored_index_files import LoadedOracle, key_range, lowest, write_scored_index_dir

EMPTY = 0xFFFFFFFF


def key_to_bits(metric, key):   # inverse of order_key (common.cuh)
    key = np.asarray(key, np.uint32)
    if metric in (1, 2):
        key = ~key
    return np.where(key & 0x80000000, key & 0x7FFFFFFF, ~key).astype(np.uint32)


def py_lowest(adj, keys, min_key, max_key):
    """ProbNode::new_with_neighbors_and_versions (prob_node.rs:155-169)"""
    li, lk = 0, max_key
    for s, (a, k) in enumerate(zip(adj, keys)):
        if a == EMPTY:
            return s, min_key
        if k < lk:
            li, lk = s, k
    return li, lk


def test_reader_returns_stored_slot_values_and_tags(tmp_path):
    vecs, mg = mdgraph.build(n=260, dim=16, md_dims=6, levels=3, nb=8, nb0=16, storage_type=4, metric=0, seed=31)
    fg = mg.fg
    rng = np.random.default_rng(5)
    scores = [rng.normal(size=a.size).astype(np.float32) for a in fg.adj]
    scores[0][:5] = np.array([-0.0, np.inf, -1.0, 2.0, np.nan], np.float32)   # odd values travel as bits
    g = dict(num_levels=fg.num_levels, neighbors_count=8, level0_neighbors_count=16, entry=fg.entry, node_row=fg.node_row,
             adj=fg.adj, child=fg.child)
    d = str(tmp_path / "idx")
    root_link, pseudo_link = write_scored_index_dir(d, 4, fg.dim, fg.codes, fg.mags, g, mg.node_id, mg.node_md, mg.md_bits, mg.md_mags,
                                                    scores, 4, pseudo_entry=mg.pseudo_entry, seed=3)
    hf = cdb.HnswFiles(d, root_link, pseudo_link)
    filled_seen = 0
    for lv in range(fg.num_levels + 1):
        nb = fg.nbrs(lv)
        src = {int(mg.node_id[lv][i]): i for i in range(fg.cnt[lv])}
        assert hf.slot_scores[lv].shape == hf.adj[lv].shape == hf.slot_tags[lv].shape
        for j, nid in enumerate(hf.node_id[lv].tolist()):
            i = src[nid]
            for s in range(nb):
                got_s, got_t = hf.slot_scores[lv][j * nb + s], hf.slot_tags[lv][j * nb + s]
                if hf.adj[lv][j * nb + s] == EMPTY:
                    assert got_t == 0xFF and got_s.view(np.uint32) == 0
                else:
                    assert got_t == 4 and got_s.view(np.uint32) == scores[lv][i * nb + s].view(np.uint32)
                    filled_seen += 1
    assert filled_seen > 1000
    hf.close()
    # damage: a truncated index file fails exactly as before
    for fid in (0, 1):
        p = os.path.join(d, f"{fid}.index")
        blob = open(p, "rb").read()
        open(p, "wb").write(blob[: len(blob) // 2])
    with pytest.raises(cdb.CosdataError):
        cdb.HnswFiles(d, root_link, pseudo_link)


@pytest.mark.parametrize("metric,st", [(0, 4), (3, 3), (1, 4)])
def test_lowest_index_rule(metric, st):
    lo, hi = key_range(metric)
    rng = np.random.default_rng(metric)
    cases = [
        ([1, 2, 3, 4], [50, 40, 40, 60]),                          # a tie: the first of the lowest
        ([1, 2, 3, 4], [hi, hi, hi, hi]),                          # every slot at MetricResult::max: slot 0, max
        ([1, 2, 3, 4], [hi, 70, hi, 70]),
        ([1, EMPTY, 3, EMPTY], [5, 0, 1, 0]),                      # the first empty slot, MetricResult::min
        ([EMPTY] * 4, [0] * 4),
        ([1, 2, 3, 4], [lo, 9, lo, 3]),                            # MetricResult::min stored in a filled slot
    ]
    for _ in range(200):
        n = int(rng.integers(1, 65))
        adj = np.where(rng.random(n) < 0.1, EMPTY, 1).astype(np.uint32)
        keys = rng.choice(np.array([lo, hi, 100, 200, 300], np.uint32), n)
        cases.append((adj, keys))
    for adj, keys in cases:
        assert lowest(adj, keys, metric) == py_lowest(list(adj), [int(k) for k in keys], lo, hi), (adj, keys)


@pytest.mark.parametrize("st,metric", [(1, 0), (3, 3)])
def test_reload_gives_back_the_build(st, metric):
    levels, nb, nb0, efc = 3, 4, 8, 24
    n, dim = 160, 16
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=3)
    root = np.linspace(-0.9, 0.9, dim).astype(np.float32)
    codes, mags = orc.quantize_batch(st, np.concatenate([pop["vecs"], root[None], np.zeros((1, dim), np.float32)]))
    o = pydelete_md.Graph(metric, st, dim, codes, mags, pop["md_bits"], pop["md_mags"], levels, nb, nb0, n, pop["main_root_md"], n + 1,
                          pop["pseudo_root_md"])
    o.insert(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], efc)
    e = o.export()
    scores = [np.where(a == EMPTY, 0, key_to_bits(metric, k)).astype(np.uint32).view(np.float32) for a, k in zip(e["adj"], e["simkey"])]
    r = LoadedOracle(metric, st, dim, codes, mags, pop["md_bits"], pop["md_mags"], levels, nb, nb0, e["node_row"], e["node_id"],
                     e["node_md"], e["adj"], e["child"], scores)
    f = r.export()
    lo, hi = key_range(metric)
    stale = 0
    for lv in range(levels + 1):
        for key in ("node_row", "node_id", "node_md", "adj") + (("child",) if lv else ()):
            assert np.array_equal(e[key][lv], f[key][lv]), (key, lv)
        filled = e["adj"][lv] != EMPTY
        assert np.array_equal(e["simkey"][lv][filled], f["simkey"][lv][filled]), lv
        nbc = nb0 if lv == 0 else nb
        for i in range(e["node_row"][lv].size):
            want = py_lowest(list(f["adj"][lv][i * nbc:(i + 1) * nbc]), list(f["simkey"][lv][i * nbc:(i + 1) * nbc]), lo, hi)
            assert (f["lowest_idx"][lv][i], f["lowest_key"][lv][i]) == want, (lv, i)
            stale += (e["lowest_idx"][lv][i], e["lowest_key"][lv][i]) != want
        # list positions: a loaded node's level-0 index, carried up; the roots have none
        ins = f["ins"][lv]
        assert ins[0] == EMPTY and ins[1] == EMPTY
        want_ins = np.arange(ins.size) if lv == 0 else f["ins"][lv - 1][f["child"][lv]]
        assert np.array_equal(ins[2:], want_ins[2:])
    assert stale > 0                                                       # the reload derives what the builder left stale
    # deleting rows from the reloaded state unlinks every node of theirs
    assert r.delete([3, 7]).tolist() == [0, 0]
    f = r.export()
    for lv in range(levels + 1):
        a = f["adj"][lv]
        assert not np.isin(f["node_row"][lv][a[a != EMPTY]], [3, 7]).any(), lv
    r.close(); o.close()


@pytest.mark.parametrize("st,metric", [(1, 0), (3, 3)])
def test_reload_without_a_pseudo_root_equals_the_plain_oracles(st, metric):
    """a collection without a metadata schema: the reload of a plain graph (node ids = rows, the root u32::MAX, no pseudo
    root) continued with inserts and deletes one at a time equals the plain insert and delete oracles on the same graph"""
    from tests import pydelete
    n0, n1, dim, levels, nb, nb0, efc, seed = 300, 120, 16, 3, 4, 8, 24, 2
    vecs = orc.synth_matrix(41, n0 + 1 + n1, dim)
    codes, mags = orc.quantize_batch(st, vecs)                             # row n0 is the root
    p = pydelete.Graph.init(metric, st, dim, codes, mags, n0, levels, nb, nb0)
    p.insert(0, n0, ef_construction=efc, seed=seed)
    e = p.export()
    ids = [np.where(a == n0, EMPTY, a).astype(np.uint32) for a in e["node_row"]]
    mds = [np.full(a.size, EMPTY, np.uint32) for a in e["node_row"]]
    scores = [np.where(a == EMPTY, 0, key_to_bits(metric, k)).astype(np.uint32).view(np.float32) for a, k in zip(e["adj"], e["simkey"])]
    r = LoadedOracle(metric, st, dim, codes, mags, np.zeros((1, 1), np.int32), np.zeros(1, np.float32), levels, nb, nb0, e["node_row"],
                     ids, mds, e["adj"], e["child"], scores, entry=e["entry"], pseudo_entry=None)
    f = r.export()
    lo, hi = key_range(metric)
    for lv in range(levels + 1):
        for key in ("node_row", "node_id", "adj") + (("child",) if lv else ()):
            want = ids[lv] if key == "node_id" else e[key][lv]
            assert np.array_equal(f[key][lv], want), (key, lv)
        nbc = nb0 if lv == 0 else nb
        for i in range(e["node_row"][lv].size):
            assert (f["lowest_idx"][lv][i], f["lowest_key"][lv][i]) == py_lowest(
                list(e["adj"][lv][i * nbc:(i + 1) * nbc]), list(e["simkey"][lv][i * nbc:(i + 1) * nbc]), lo, hi), (lv, i)
    with pytest.raises(ValueError):                                        # no pseudo root: no pseudo replicas
        r.insert([EMPTY], [5], [5], [EMPTY], [0], efc)
    # the plain oracles on the same graph (symmetric arms: the recomputed similarities are the stored ones)
    q = pydelete.Graph.from_graph(metric, st, dim, codes, mags, p.export())
    draws = np.random.default_rng(3).integers(0, 2, n1).astype(np.uint8)
    new = np.arange(n0 + 1, n0 + 1 + n1, dtype=np.uint32)
    assert np.array_equal(q.insert(n0 + 1, n1, ef_construction=efc, max_level=draws),
                          r.insert(new, new, new, np.full(n1, EMPTY, np.uint32), draws, efc))
    dead = np.random.default_rng(4).choice(np.concatenate([np.arange(n0), new]), 40, replace=False).astype(np.uint32)
    assert np.array_equal(q.delete(dead), r.delete(dead))
    e, f = q.export(), r.export()
    for lv in range(levels + 1):
        for key in ("node_row", "adj", "simkey", "lowest_idx", "lowest_key") + (("child",) if lv else ()):
            assert np.array_equal(f[key][lv], e[key][lv]), (key, lv)
    r.close(); q.close(); p.close()
