"""CDB_MODE_HNSW parity: the CUDA search on an uploaded flat graph must reproduce the oracle's
search_internal (ann_search + remove_duplicates_and_filter + exact re-rank) on the SAME graph:
ids, scores (bit-identical), counts, error flags and even the number of distance evaluations."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from oracle import pyhnsw

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def clustered(n, dim, seed):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(32, dim)).astype(np.float32)
    v = (centres[rng.integers(0, 32, n)] + 0.35 * rng.normal(size=(n, dim))).astype(np.float32)
    return (v / (np.abs(v).max() * 1.01)).astype(np.float32)


def build_both(vecs, st, metric, levels=5, nb=16, nb0=32, efc=64, seed=5):
    n, dim = vecs.shape
    root = orc.synth_matrix(31337, 1, dim)[0]
    fg = pyhnsw.build(int(metric), int(st), vecs, root, num_levels=levels, neighbors_count=nb,
                      level0_neighbors_count=nb0, ef_construction=efc, seed=seed)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(np.concatenate([vecs, root[None]], axis=0))          # root vector is the last row (row n)
    codes, mags = ix.read_codes(0, n + 1)
    assert np.array_equal(codes, fg.codes) and np.array_equal(bits(mags), bits(fg.mags))
    ix.set_graph(levels, nb, nb0, fg.entry, n, fg.node_row, fg.adj, fg.child)
    return fg, ix


@pytest.mark.parametrize("st,metric", [(ST.HalfPrecisionFP, MK.Cosine), (ST.UnsignedByte, MK.Cosine),
                                        (ST.SubByte2, MK.DotProduct), (ST.FullPrecisionFP, MK.Cosine),
                                        (ST.SubByte3, MK.Cosine), (ST.HalfPrecisionFP, MK.DotProduct),
                                        (ST.BFloat16, MK.Cosine), (ST.BFloat16, MK.DotProduct)])
@pytest.mark.parametrize("ef", [16, 64, 256])
def test_hnsw_search_matches_oracle(st, metric, ef):
    n, dim, k = 2500, 48, 10
    vecs = clustered(n, dim, 1)
    fg, ix = build_both(vecs, st, metric)
    rng = np.random.default_rng(2)
    queries = (vecs[rng.integers(0, n, 33)] + 0.05 * rng.normal(size=(33, dim))).astype(np.float32)
    ev0, pp0 = ix.hnsw_counters()
    ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=64)
    ev1, pp1 = ix.hnsw_counters()
    want_ids, want_scores, want_counts, want_err, ev, pp = pyhnsw.search_batch(fg, vecs, queries, k, ef_search=ef)
    assert np.array_equal(err, want_err)
    assert np.array_equal(counts, want_counts)
    assert np.array_equal(ids, want_ids)
    assert np.array_equal(bits(scores), bits(want_scores))
    assert (ev1 - ev0, pp1 - pp0) == (ev, pp)            # same traversal, node for node
    ix.close()


@pytest.mark.parametrize("flags,name", [(0, "plain"), (2, "preload"), (4, "atomic fixed set"), (22, "pool + arg-max pops"), (38, "speculative scoring"), (32, "speculative, plain"), (8, "cta per query")])
@pytest.mark.parametrize("st,ef,nb0", [(ST.HalfPrecisionFP, 128, 32), (ST.HalfPrecisionFP, 300, 64), (ST.UnsignedByte, 40, 32),
                                       (ST.BFloat16, 64, 64)])
def test_hnsw_kernel_variants_walk_the_same_path(flags, name, st, ef, nb0):
    # the search kernel must pop the same nodes in the same order as the oracle (ef 300: not a power of two, EFP 512; nb0 64:
    # the second slot per lane), and every value cdb_debug_set_hnsw_flags accepts must give the default's arrays and counters:
    # none of these values selects anything on a plain graph
    n, dim, k = 3000, 40, 10
    vecs = clustered(n, dim, 21)
    fg, ix = build_both(vecs, st, MK.Cosine, levels=4, nb=16, nb0=nb0, efc=48, seed=3)
    rng = np.random.default_rng(22)
    queries = (vecs[rng.integers(0, n, 70)] + 0.05 * rng.normal(size=(70, dim))).astype(np.float32)
    want = pyhnsw.search_batch(fg, vecs, queries, k, ef_search=ef)

    def search(fl):
        try:
            cdb.debug_set_hnsw_flags(fl)
            ev0, pp0 = ix.hnsw_counters()
            ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=64)
            ev1, pp1 = ix.hnsw_counters()
        finally:
            cdb.debug_set_hnsw_flags()
        return ids, bits(scores), counts, err, np.array([ev1 - ev0, pp1 - pp0])

    ids, scores, counts, err, evpp = search(0xFFFFFFFF)
    assert np.array_equal(ids, want[0]) and np.array_equal(scores, bits(want[1]))
    assert np.array_equal(counts, want[2]) and np.array_equal(err, want[3])
    assert tuple(evpp) == (want[4], want[5])
    for got, default in zip(search(flags), (ids, scores, counts, err, evpp)):
        assert np.array_equal(got, default), name
    ix.close()


def test_hnsw_pool_trims_and_exact_selections_walk_the_same_path():
    # ef = EFP = 128 and 64 level-0 slots over spread-out rows: the first pops bring up to 64 new candidates each, so the pool
    # (2 * EFP entries) fills while R, the pops still to come, is close to ef.  Then the pool is trimmed, and some trims find
    # no sampled pivot with between R and 2 * EFP - 64 better entries and fall back to the exact selection.  The pop order
    # must stay the oracle's, in the plain kernel and in the instrumented one that counts both events.
    n, dim, k, ef = 5000, 40, 10, 128
    vecs = np.random.default_rng(21).uniform(-0.9, 0.9, size=(n, dim)).astype(np.float32)
    fg, ix = build_both(vecs, ST.HalfPrecisionFP, MK.Cosine, levels=4, nb=16, nb0=64, efc=48, seed=3)
    rng = np.random.default_rng(22)
    queries = (vecs[rng.integers(0, n, 500)] + 0.05 * rng.normal(size=(500, dim))).astype(np.float32)
    want = pyhnsw.search_batch(fg, vecs, queries, k, ef_search=ef)
    for profile in (False, True):
        if profile:
            ix.hnsw_profile(enable=True, read=False)
        ev0, pp0 = ix.hnsw_counters()
        ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=64)
        ev1, pp1 = ix.hnsw_counters()
        assert np.array_equal(ids, want[0]) and np.array_equal(bits(scores), bits(want[1]))
        assert np.array_equal(counts, want[2]) and np.array_equal(err, want[3])
        assert (ev1 - ev0, pp1 - pp0) == (want[4], want[5])
    prof = ix.hnsw_profile(enable=False, read=True)
    assert prof["trims"] > 0 and prof["exact_selections"] > 0, prof
    ix.close()


def test_hnsw_default_params_recall_and_shortlist():
    # reference defaults (config.toml:19-33): nbrs 32/64, ef_search 256, shortlist 64, 9 layers
    n, dim, k = 4000, 64, 10
    vecs = clustered(n, dim, 7)
    fg, ix = build_both(vecs, ST.HalfPrecisionFP, MK.Cosine, levels=9, nb=32, nb0=64, efc=128, seed=9)
    rng = np.random.default_rng(8)
    queries = (vecs[rng.integers(0, n, 64)] + 0.05 * rng.normal(size=(64, dim))).astype(np.float32)
    for shortlist in (64, 16):
        ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=256, shortlist_size=shortlist)
        w = pyhnsw.search_batch(fg, vecs, queries, k, ef_search=256, shortlist_size=shortlist)
        assert np.array_equal(ids, w[0]) and np.array_equal(bits(scores), bits(w[1]))
    gt, _ = orc.brute_topk_f32(vecs, queries, k)
    recall = np.mean([len(set(ids[i]) & set(gt[i])) / k for i in range(len(queries))])
    assert recall >= 0.80, recall                                   # and equal to the oracle's by construction
    ix.close()


@pytest.mark.parametrize("flags", [None, 38, 22])
def test_hnsw_zero_norm_row_fails_the_query_like_the_reference(flags):
    # a row whose norm is 0 is a CalculationError the moment a traversal scores it (cosine.rs:230-231): exactly the queries that
    # reach it fail.  The graph is built over normal vectors (an insert that errors is not indexed at all), then the stored vector
    # of one well-connected node is replaced by zeros.  flags 38 and 22: values that once selected speculative scoring and the
    # unsorted candidate pool, still accepted and now running the default form.
    n, dim, k = 1500, 32, 5
    vecs = clustered(n, dim, 3)
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    root = orc.synth_matrix(31337, 1, dim)[0]
    fg = pyhnsw.build(int(metric), int(st), vecs, root, num_levels=5, neighbors_count=16, level0_neighbors_count=32,
                      ef_construction=64, seed=5)
    hub = int(np.bincount(fg.adj[0][fg.adj[0] < n], minlength=n).argmax())      # the most linked-to data row
    stored = vecs.copy()
    stored[hub] = 0.0
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(np.concatenate([stored, root[None]], axis=0))
    ix.set_graph(5, 16, 32, fg.entry, n, fg.node_row, fg.adj, fg.child)
    codes, mags = ix.read_codes(0, n + 1)
    fz = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n, 5, 16, 32, fg.entry, fg.node_row, fg.adj, fg.child)
    rng = np.random.default_rng(5)
    near = vecs[hub] + 0.02 * rng.normal(size=(6, dim)).astype(np.float32)
    queries = np.concatenate([near, vecs[rng.integers(0, n, 60)] + 0.02]).astype(np.float32)
    try:
        if flags is not None:
            cdb.debug_set_hnsw_flags(flags)
        ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=24, shortlist_size=64)
    finally:
        cdb.debug_set_hnsw_flags()
    w = pyhnsw.search_batch(fz, stored, queries, k, ef_search=24)
    assert 0 < (w[3] != 0).sum() < len(queries)                       # some traversals reach the zero row, others do not
    assert np.array_equal(err, w[3]) and np.array_equal(counts, w[2])
    assert np.array_equal(ids, w[0]) and np.array_equal(bits(scores), bits(w[1]))
    ix.close()


def test_hnsw_requires_graph_and_valid_params():
    ix = cdb.DenseIndex(dim=16, capacity=10, keep_raw_f32=True, storage_type=ST.HalfPrecisionFP)
    ix.append(orc.synth_matrix(1, 10, 16))
    with pytest.raises(cdb.CosdataError) as e:
        ix.batch_search(orc.synth_matrix(2, 1, 16), 3, cdb.SearchMode.HNSW)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    ix.close()
