"""HNSW at production row sizes (D = 768 .. 12288): the traversal against its oracles where a pop's neighbours no longer fit
one staging group.

The traversal (hw_traverse_level, hnsw_traverse.cuh: the searches, the build, the insert and the delete's phase A) scores a
pop's accepted neighbours in groups of staged rows, copied with TMA bulk copies that complete on the warp's mbarrier, one
phase per group.  At D <= 64 every pop fits one group; at D = 768 a group holds about a dozen rows, so with 64 level-0
neighbours a pop runs several groups and the first Err may sit in a later one.  D = 769 reaches the scalar tail of the f16 dot chain.
Every comparison is exact: ids, score bits, counts, error flags, evaluation and pop counts, graphs array for array.
The graph writers refuse an ef whose shared memory exceeds the device's limit before anything changes."""
import ctypes as C
import functools

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from oracle import pyhnsw, pymeta
from tests import mdgraph, pydelete, pyinsert

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
EMPTY = 0xFFFFFFFF
LEVELS, NB, NB0, SHORTLIST = 4, 16, 64, 64


# ----------------------------------------------------------------------------- staged rows per group, restated
def round16(x):
    return (x + 15) // 16 * 16


def row_pitch(st, dim):   # common.cuh row_pitch_bytes
    if st == ST.UnsignedByte:
        return round16(dim)
    if st in (ST.SubByte1, ST.SubByte2, ST.SubByte3):
        return int(st) * round16((dim + 7) // 8)
    return round16(dim * (4 if st == ST.FullPrecisionFP else 2))


def stage_pitch(pitch):
    return round16(pitch) + 16


def stage_rows(pitch):   # hw_carve: 18700 B, at most one row per lane
    return min(32, max(1, 18700 // stage_pitch(pitch)))


def carve_bytes(pitch, ef):   # hw_carve(pitch, ef).total: the traversal's dynamic shared memory (plain graphs, writers)
    efp = max(128, 1 << max(0, (ef - 1).bit_length()))
    # query row, qkeys [2 EFP], rkeys [EFP], nkeys [64], mbarrier, fixed set [128 words], qnodes [2 EFP], rnodes [EFP], nnodes, nrow
    base = round16(pitch) + (3 * efp + 64) * 8 + 8 + 128 * 4 + (3 * efp + 2 * 64) * 4
    return round16(base) + stage_rows(pitch) * stage_pitch(pitch)


# (storage, metric, D) -> rows per group
SHAPES = {
    (ST.HalfPrecisionFP, MK.Cosine, 768): 12,
    (ST.HalfPrecisionFP, MK.DotProduct, 768): 12,
    (ST.BFloat16, MK.Cosine, 768): 12,
    (ST.HalfPrecisionFP, MK.Cosine, 769): 11,
    (ST.HalfPrecisionFP, MK.Cosine, 1000): 9,
    (ST.FullPrecisionFP, MK.Cosine, 768): 6,
    (ST.UnsignedByte, MK.Cosine, 768): 23,
    (ST.SubByte3, MK.Cosine, 1000): 32,
    (ST.SubByte2, MK.Cosine, 4096): 17,
    (ST.SubByte2, MK.DotProduct, 4096): 17,
    (ST.FullPrecisionFP, MK.Cosine, 4096): 1,
}


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def clustered(n, dim, seed):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(32, dim)).astype(np.float32)
    v = (centres[rng.integers(0, 32, n)] + 0.35 * rng.normal(size=(n, dim))).astype(np.float32)
    return (v / (np.abs(v).max() * 1.01)).astype(np.float32)


def near(vecs, nq, seed, noise=0.05):
    rng = np.random.default_rng(seed)
    return (vecs[rng.integers(0, vecs.shape[0], nq)] + noise * rng.normal(size=(nq, vecs.shape[1]))).astype(np.float32)


def root_vector(seed, dim, lo=-1.0, hi=1.0):   # the root the build appends
    s = orc.synth(seed ^ 0x526F6F74, 0, dim)
    return (np.float32(lo) + (s + np.float32(1.0)) * np.float32(0.5) * np.float32(hi - lo)).astype(np.float32)


@functools.lru_cache(maxsize=None)
def oracle_graph(st, metric, dim, n=1500, seed=1):
    """clustered rows and the oracle builder's graph over them (root = row n), shared by the search cases"""
    vecs = clustered(n, dim, seed)
    root = orc.synth_matrix(31337, 1, dim)[0]
    fg = pyhnsw.build(int(metric), int(st), vecs, root, num_levels=LEVELS, neighbors_count=NB, level0_neighbors_count=NB0,
                      ef_construction=64, seed=5)
    return vecs, root, fg


def upload(stored, root, fg, st, metric):
    n, dim = stored.shape
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(np.concatenate([stored, root[None]]))
    ix.set_graph(LEVELS, NB, NB0, fg.entry, n, fg.node_row, fg.adj, fg.child)
    return ix


def gpu_search(ix, queries, k, ef):
    ev0, pp0 = ix.hnsw_counters()
    ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=SHORTLIST)
    ev1, pp1 = ix.hnsw_counters()
    return ids, scores, counts, err, ev1 - ev0, pp1 - pp0


def assert_search_equal(got, want, what):
    ids, scores, counts, err, ev, pp = got
    assert np.array_equal(err, want[3]), what
    assert np.array_equal(counts, want[2]), what
    assert np.array_equal(ids, want[0]), what
    assert np.array_equal(bits(scores), bits(want[1])), what
    assert (ev, pp) == (want[4], want[5]), what


def assert_graph_equal(g, e, scores, metric):
    assert g["entry"] == e["entry"] and g["root_row"] == e["root_row"]
    for lv in range(g["num_levels"] + 1):
        assert np.array_equal(g["node_row"][lv], e["node_row"][lv]), lv
        assert np.array_equal(g["adj"][lv], e["adj"][lv]), lv
        if lv:
            assert np.array_equal(g["child"][lv], e["child"][lv]), lv
        assert np.array_equal(bits(scores[lv]), bits(pyinsert.slot_scores(metric, e["simkey"][lv], e["adj"][lv]))), lv


def nodes_over(adj0, rows):
    """level-0 nodes that link more neighbours than one group of `rows` staged rows holds"""
    return int(((np.asarray(adj0).reshape(-1, NB0) != EMPTY).sum(1) > rows).sum())


# ----------------------------------------------------------------------------- 1. search on an uploaded oracle graph
@pytest.mark.parametrize("st,metric,dim", list(SHAPES), ids=[f"{s.name}-{m.name}-{d}" for s, m, d in SHAPES])
def test_search_variants_at_production_row_sizes(st, metric, dim):
    pitch = row_pitch(st, dim)
    rows = stage_rows(pitch)
    assert rows == SHAPES[(st, metric, dim)]
    assert rows < NB0                              # a pop can score more neighbours than one group holds
    vecs, root, fg = oracle_graph(st, metric, dim)
    n = vecs.shape[0]
    ix = upload(vecs, root, fg, st, metric)
    codes, mags = ix.read_codes(0, n + 1)
    assert np.array_equal(codes, fg.codes) and np.array_equal(bits(mags), bits(fg.mags))
    assert nodes_over(fg.adj[0], rows) > n // 4
    nq = 130 if (st, metric, dim) == (ST.HalfPrecisionFP, MK.Cosine, 768) else 64
    queries = near(vecs, nq, 2)
    k = 10
    for ef in (64, 300):
        want = pyhnsw.search_batch(fg, vecs, queries, k, ef_search=ef)
        assert (want[3] == 0).all() and (want[2] == k).all()
        assert_search_equal(gpu_search(ix, queries, k, ef), want, ef)
    ix.close()


# ----------------------------------------------------------------------------- 2. the first Err in a later group
@pytest.mark.parametrize("st,dim", [(ST.HalfPrecisionFP, 768), (ST.FullPrecisionFP, 4096)])
def test_zero_norm_hub_fails_the_queries_that_reach_it(st, dim):
    # the stored vector of the most linked-to row is replaced by zeros after the build: a traversal that scores it returns a
    # CalculationError, and the pop's earlier evaluations must not hide it (f32 x 4096: one row per group)
    metric = MK.Cosine
    vecs, root, fg = oracle_graph(st, metric, dim)
    n = vecs.shape[0]
    hub = int(np.bincount(fg.adj[0][fg.adj[0] < n], minlength=n).argmax())
    stored = vecs.copy()
    stored[hub] = 0.0
    ix = upload(stored, root, fg, st, metric)
    codes, mags = ix.read_codes(0, n + 1)
    fz = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n, LEVELS, NB, NB0, fg.entry, fg.node_row, fg.adj, fg.child)
    rng = np.random.default_rng(5)
    queries = np.concatenate([vecs[hub] + 0.02 * rng.normal(size=(6, dim)), near(vecs, 90, 6, 0.02)]).astype(np.float32)
    k, ef = 5, 8
    want = pyhnsw.search_batch(fz, stored, queries, k, ef_search=ef)
    assert 0 < (want[3] != 0).sum() < len(queries)                      # some traversals reach the zero row, others do not
    ids, scores, counts, err, _, _ = gpu_search(ix, queries, k, ef)
    assert np.array_equal(err, want[3]) and np.array_equal(counts, want[2])
    assert np.array_equal(ids, want[0]) and np.array_equal(bits(scores), bits(want[1]))
    ok = np.flatnonzero(want[3] == 0)                                   # error-free traversals: node for node
    w_ok = pyhnsw.search_batch(fz, stored, queries[ok], k, ef_search=ef)
    assert_search_equal(gpu_search(ix, queries[ok], k, ef), w_ok, "error-free queries")
    ix.close()


# ----------------------------------------------------------------------------- 3. sequential build == oracle builder
@pytest.mark.parametrize("st,metric,dim", [(ST.HalfPrecisionFP, MK.Cosine, 768), (ST.BFloat16, MK.DotProduct, 769),
                                           (ST.UnsignedByte, MK.Cosine, 768), (ST.FullPrecisionFP, MK.Cosine, 768),
                                           (ST.SubByte3, MK.Cosine, 1000)])
def test_sequential_build_equals_oracle_builder(st, metric, dim):
    n, efc, seed = 1200, 48, 5
    vecs = clustered(n, dim, 11)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(LEVELS, NB, NB0, efc, SHORTLIST, 1, seed)
    g, sc = ix.read_graph(), ix.read_graph_slot_scores()
    codes, mags = ix.read_codes(0, n + 1)
    rc, rm = orc.quantize_batch(int(st), root_vector(seed, dim)[None])
    assert np.array_equal(codes[n], rc[0]) and bits(mags[n]) == bits(rm[0])
    o = pyinsert.Graph.init(int(metric), int(st), dim, codes, mags, n, LEVELS, NB, NB0)
    assert o.insert(0, n, ef_construction=efc, seed=seed).sum() == 0
    assert_graph_equal(g, o.export(), sc, int(metric))
    assert nodes_over(g["adj"][0], stage_rows(row_pitch(st, dim))) > n // 4
    o.close()
    ix.close()


# ----------------------------------------------------------------------------- 4. sequential insert and delete
def test_sequential_insert_equals_oracle_after_build_and_after_upload():
    st, metric, dim = ST.HalfPrecisionFP, MK.Cosine, 768
    n0, efc, seed = 800, 48, 5
    vecs = clustered(n0 + 300, dim, 13)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 301, keep_raw_f32=True)
    ix.append(vecs[:n0])
    ix.build_graph(LEVELS, NB, NB0, efc, SHORTLIST, 1, seed)
    g0 = ix.read_graph()
    for first, c in ((n0, 200), (n0 + 200, 100)):
        ix.append(vecs[first:first + c])
        failed = ix.insert_graph(efc, SHORTLIST, 1, seed)
        assert failed.size == c and failed.sum() == 0
    g, sc = ix.read_graph(), ix.read_graph_slot_scores()
    codes, mags = ix.read_codes(0, n0 + 301)
    o = pyinsert.Graph.init(int(metric), int(st), dim, codes, mags, n0, LEVELS, NB, NB0)
    o.insert(0, n0, ef_construction=efc, seed=seed)
    o.insert(n0 + 1, 200, ef_construction=efc, seed=seed)
    o.insert(n0 + 201, 100, ef_construction=efc, seed=seed)
    assert_graph_equal(g, o.export(), sc, int(metric))
    # the same rows inserted into the uploaded first build (slot state derived on upload)
    up = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 301, keep_raw_f32=True)
    up.append(np.concatenate([vecs[:n0], root_vector(seed, dim)[None], vecs[n0:]]))
    up.set_graph(g0["num_levels"], NB, NB0, g0["entry"], g0["root_row"], g0["node_row"], g0["adj"], g0["child"])
    failed = up.insert_graph(efc, SHORTLIST, 1, seed)
    assert failed.size == 300 and failed.sum() == 0
    ou = pyinsert.Graph.from_graph(int(metric), int(st), dim, codes, mags, g0)
    ou.insert(n0 + 1, 300, ef_construction=efc, seed=seed)
    assert_graph_equal(up.read_graph(), ou.export(), up.read_graph_slot_scores(), int(metric))
    for x in (ix, up, o, ou):
        x.close()


@pytest.mark.parametrize("st", [ST.HalfPrecisionFP, ST.UnsignedByte])
def test_sequential_delete_equals_oracle(st):
    # a delete traverses with ef 512: a long queue and multi-group pops on every level
    metric, dim, n0, efc, seed = MK.Cosine, 768, 900, 48, 5
    vecs = clustered(n0, dim, 17)
    # a zero-norm row (u8: every code 0, the low end of the value range): its insert fails (unlinked); its delete fails its
    # traversal: status 2
    vecs[7] = 0.0 if st == ST.HalfPrecisionFP else -1.0
    rows = np.concatenate([[7], np.random.default_rng(3).choice(np.arange(8, n0), 40, replace=False), [7]]).astype(np.uint32)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(LEVELS, NB, NB0, efc, SHORTLIST, 1, seed)
    codes, mags = ix.read_codes(0, n0 + 1)
    status = ix.delete_rows(rows, SHORTLIST, 1)
    o = pydelete.Graph.init(int(metric), int(st), dim, codes, mags, n0, LEVELS, NB, NB0)
    failed = o.insert(0, n0, ef_construction=efc, seed=seed)
    want = o.delete(rows)
    assert np.array_equal(status, want)
    assert mags[7] == 0 and failed[7] != 0 and status[0] == 2 and status[-1] == 1
    assert_graph_equal(ix.read_graph(), o.export(), ix.read_graph_slot_scores(), int(metric))
    assert np.array_equal(np.flatnonzero(ix.deleted_rows()), np.unique(rows))
    ix.close()
    o.close()


# ----------------------------------------------------------------------------- 5. filtered search
@pytest.mark.parametrize("st", [ST.HalfPrecisionFP, ST.FullPrecisionFP])
def test_filtered_search_matches_oracle(st):
    metric, dim, k, ef = MK.Cosine, 768, 10, 64
    vecs, mg = mdgraph.build(n=1000, dim=dim, md_dims=7, levels=LEVELS, nb=NB, nb0=NB0, storage_type=int(st), metric=int(metric),
                             seed=21)
    q, filters = mdgraph.make_queries(vecs, mg, 96, seed=9)
    fg = mg.fg
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=vecs.shape[0], keep_raw_f32=True)
    ix.append(vecs)
    ix.set_graph(fg.num_levels, fg.neighbors_count, fg.level0_neighbors_count, fg.entry, fg.n, fg.node_row, fg.adj, fg.child)
    ix.set_graph_metadata(mg.md_bits, mg.md_mags, mg.node_id, mg.node_md, mg.pseudo_entry)
    ids, scores, counts, err = ix.batch_search_filtered(q, filters, k, ef_search=ef, shortlist_size=SHORTLIST)
    want = pymeta.search_batch_md(mg, vecs, q, filters, k, ef_search=ef)
    assert np.array_equal(err, want[3]) and np.array_equal(counts, want[2])
    assert np.array_equal(ids, want[0]) and np.array_equal(bits(scores), bits(want[1]))
    assert (want[2] > 0).sum() > len(q) // 2
    sel = np.flatnonzero(want[3] == 0)                                   # error-free queries: node for node
    ev0, pp0 = ix.hnsw_counters()
    ix.batch_search_filtered(q[sel], [filters[i] for i in sel], k, ef_search=ef, shortlist_size=SHORTLIST)
    ev1, pp1 = ix.hnsw_counters()
    w = pymeta.search_batch_md(mg, vecs, q[sel], [filters[i] for i in sel], k, ef_search=ef)
    assert (ev1 - ev0, pp1 - pp0) == (w[4], w[5])
    ix.close()


# ----------------------------------------------------------------------------- 6. the headline shape at reduced N
def test_batched_build_at_250k_f16_768_search_parity_and_recall():
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 8 << 30:
        pytest.skip(f"needs 8 GB of free device memory, {free >> 20} MB free")
    n, dim, nq, k, ef = 250_000, 768, 512, 10, 128
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    # bench.py's c3 mixture at the same number of rows per centre (about 244): stored rows and fresh queries
    rng = np.random.default_rng(41)
    centres = rng.normal(size=(n // 244, dim)).astype(np.float32)
    scale = np.float32(1.0 / (4.5 * 1.06))
    mix = lambda m: ((centres[rng.integers(0, len(centres), m)] + 0.35 * rng.normal(size=(m, dim)).astype(np.float32))
                     * scale).clip(-0.999, 0.999).astype(np.float32)
    vecs, queries = mix(n), mix(nq)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(LEVELS, NB, NB0, 64, SHORTLIST, seed=9)
    g = ix.read_graph()
    codes, mags = ix.read_codes(0, n + 1)
    fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n, LEVELS, NB, NB0, g["entry"], g["node_row"], g["adj"], g["child"])
    got = gpu_search(ix, queries, k, ef)
    want = pyhnsw.search_batch(fg, vecs, queries, k, ef_search=ef)
    assert_search_equal(got, want, "default flags")
    gt, _, _, _ = ix.batch_search(queries, k, cdb.SearchMode.BRUTE_RAW)   # the exact f32 scan
    recall = np.mean([len(set(got[0][i]) & set(gt[i])) / k for i in range(nq)])
    assert recall >= 0.9, recall
    ix.close()


# ----------------------------------------------------------------------------- 7. shared-memory bounds of the graph writers
@pytest.mark.parametrize("st", [ST.FullPrecisionFP, ST.HalfPrecisionFP, ST.UnsignedByte])
def test_append_magnitudes_around_the_48kb_default(st):
    # a small append computes magnitudes with one CTA per row, the squares staged in 4·D bytes of shared memory next to a
    # static word: D = 12288 fills the 48 KB default exactly, so that launch would fail; wider rows take the thread-per-row form
    for dim in (12284, 12287, 12288, 12289):
        vecs = clustered(5, dim, dim)
        ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=MK.Cosine, capacity=5)
        ix.append(vecs)
        codes, mags = ix.read_codes(0, 5)
        want_codes, want_mags = orc.quantize_batch(int(st), vecs)
        assert np.array_equal(codes, want_codes) and np.array_equal(bits(mags), bits(want_mags)), dim
        ix.close()


def optin_limit():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def test_build_insert_and_search_refuse_shapes_over_the_shared_memory_limit():
    st, metric, dim, n, seed = ST.FullPrecisionFP, MK.Cosine, 12288, 200, 3
    assert carve_bytes(row_pitch(st, dim), 4096) == 247328 > optin_limit()
    vecs = clustered(n + 20, dim, 23)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 21, keep_raw_f32=True)
    ix.append(vecs[:n])
    codes0, mags0 = ix.read_codes(0, n)
    with pytest.raises(cdb.CosdataError) as e:
        ix.build_graph(LEVELS, NB, NB0, 4096, SHORTLIST, 1, seed)
    assert e.value.status == cdb.Status.INVALID_PARAMS and "shared memory" in str(e.value)
    assert len(ix) == n                                                 # no root row appended, no graph, codes as they were
    with pytest.raises(cdb.CosdataError):
        ix.read_graph()
    codes1, mags1 = ix.read_codes(0, n)
    assert np.array_equal(codes1, codes0) and np.array_equal(bits(mags1), bits(mags0))
    # the same index builds at ef_construction 64, one row at a time equal to the oracle
    ix.build_graph(LEVELS, NB, NB0, 64, SHORTLIST, 1, seed)
    g, sc = ix.read_graph(), ix.read_graph_slot_scores()
    codes, mags = ix.read_codes(0, n + 1)
    o = pyinsert.Graph.init(int(metric), int(st), dim, codes, mags, n, LEVELS, NB, NB0)
    o.insert(0, n, ef_construction=64, seed=seed)
    assert_graph_equal(g, o.export(), sc, int(metric))
    o.close()
    # an insert at ef_construction 4096 is refused and leaves the graph and its slot state as they were
    ix.append(vecs[n:])
    with pytest.raises(cdb.CosdataError) as e:
        ix.insert_graph(4096, SHORTLIST, 1, seed)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    g1, sc1 = ix.read_graph(), ix.read_graph_slot_scores()
    for lv in range(LEVELS + 1):
        assert np.array_equal(g1["node_row"][lv], g["node_row"][lv]) and np.array_equal(g1["adj"][lv], g["adj"][lv]), lv
        assert np.array_equal(g1["child"][lv], g["child"][lv]) and np.array_equal(bits(sc1[lv]), bits(sc[lv])), lv
    assert g1["entry"] == g["entry"] and len(ix) == n + 21
    # search: ef_search 4096 is refused, ef_search 64 equals the oracle on the built graph
    queries = near(vecs[:n], 16, 4)
    with pytest.raises(cdb.CosdataError) as e:
        ix.batch_search(queries, 5, cdb.SearchMode.HNSW, ef_search=4096, shortlist_size=SHORTLIST)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n, LEVELS, NB, NB0, g["entry"], g["node_row"], g["adj"], g["child"])
    want = pyhnsw.search_batch(fg, vecs[:n], queries, 5, ef_search=64)
    assert_search_equal(gpu_search(ix, queries, 5, 64), want, "default")
    ix.close()


def test_build_above_200kb_but_under_the_limit_still_builds():
    st, metric, dim, n, seed = ST.FullPrecisionFP, MK.Cosine, 8192, 200, 4
    assert 200 * 1024 < carve_bytes(row_pitch(st, dim), 4096) == 214560 < optin_limit()
    vecs = clustered(n, dim, 29)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(LEVELS, NB, NB0, 4096, SHORTLIST, 1, seed)
    g, sc = ix.read_graph(), ix.read_graph_slot_scores()
    codes, mags = ix.read_codes(0, n + 1)
    o = pyinsert.Graph.init(int(metric), int(st), dim, codes, mags, n, LEVELS, NB, NB0)
    o.insert(0, n, ef_construction=4096, seed=seed)
    assert_graph_equal(g, o.export(), sc, int(metric))
    o.close()
    ix.close()


def test_replica_build_and_delete_refuse_shapes_over_the_shared_memory_limit():
    # the replica build checks ef_construction like the build; the delete traverses at ef 512
    pop = mdgraph.replica_population(n=40, dim=12288, md_dims=4, levels=2, seed=3)
    n, dim = pop["vecs"].shape
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.FullPrecisionFP, metric=MK.Cosine, capacity=n + 2, keep_raw_f32=True)
    ix.append(pop["vecs"])
    with pytest.raises(cdb.CosdataError) as e:
        ix.build_graph_replicas(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], pop["md_bits"],
                                pop["md_mags"], pop["main_root_md"], pop["pseudo_root_md"], 2, 8, 16, 4096, 64, 64, 1)
    assert e.value.status == cdb.Status.INVALID_PARAMS and len(ix) == n
    failed = ix.build_graph_replicas(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], pop["md_bits"],
                                     pop["md_mags"], pop["main_root_md"], pop["pseudo_root_md"], 2, 8, 16, 64, 64, 64, 1)
    assert failed.sum() == 0 and len(ix) == n + 2
    ix.close()
    # a delete traverses at ef 512, which holds the row twice (query and stage): f32 x 28672 is over the limit
    big = 28672
    assert carve_bytes(row_pitch(ST.FullPrecisionFP, big), 512) == 249376 > optin_limit()
    d = cdb.DenseIndex(dim=big, storage_type=ST.FullPrecisionFP, metric=MK.Cosine, capacity=4)
    d.append(clustered(3, big, 5))
    adj = np.array([1, EMPTY, 0, EMPTY, 0, 1], np.uint32)
    d.set_graph(0, 2, 2, 2, 2, [np.arange(3, dtype=np.uint32)], [adj], [np.zeros(3, np.uint32)])
    r = np.array([0], np.uint32)
    rc = d._lib.cdb_index_delete_rows(d._h, r.ctypes.data_as(C.c_void_p), 1, 64, 0, None, None)
    assert rc == int(cdb.Status.INVALID_PARAMS)
    assert not d.deleted_rows().any() and np.array_equal(d.read_graph()["adj"][0], adj)
    d.close()
