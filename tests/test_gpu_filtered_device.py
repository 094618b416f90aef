"""Filtered HNSW search on graphs with a metadata schema: the warp-per-query metadata kernel and the device entry point.
  * the warp kernel equals oracle/metadata_oracle.c bit for bit (ids, scores, counts, error flags, and the evaluation and pop
    counts of error-free queries) over storage types, metrics, ef, shortlists, filter shapes and D = 768 / 769;
  * the same on graphs built, grown, shrunk on the GPU and loaded from index files;
  * with edge filters at D = 768 f16 and D = 40 u8, the filtered search and the plain entry point on the same graph (every
    query unfiltered, deduplicated by replica id and re-ranked) equal the oracle;
  * cdb_search_batch_filtered_device equals the host form on caller streams, and flags bad filter ranges per query;
  * the shared-memory limit accepts ef 4096 at D = 768 f32 and refuses it at D = 8192."""
import numpy as np
import pytest
import torch

import cosdata_b200 as cdb
from oracle import pyhnsw, pymeta
from tests import mdgraph
from tests.test_gpu_hnsw_insert_replicas import build_a, full_table, grown_population, insert_b
from tests.test_gpu_hnsw_loaded_graph import cold_start

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
BAD_FILTER = 8


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def with_edge_filters(q, filters, md_dims):
    """adds Some([]), an all-zero row and 4 / 5 rows with duplicates to the filters of make_queries"""
    filters = list(filters)
    rng = np.random.default_rng(5)
    filters[1] = []
    filters[2] = [np.zeros(md_dims, np.int8)]
    row = rng.integers(0, 2, md_dims).astype(np.int8)
    filters[3] = [row, row, rng.integers(-1, 2, md_dims).astype(np.int8), row]
    filters[7] = [row, rng.integers(0, 2, md_dims).astype(np.int8), row, rng.integers(0, 2, md_dims).astype(np.int8), row]
    return q, filters


def md_index(vecs, mg, st, metric):
    fg = mg.fg
    ix = cdb.DenseIndex(dim=vecs.shape[1], storage_type=st, metric=metric, capacity=vecs.shape[0], keep_raw_f32=True)
    ix.append(vecs)
    ix.set_graph(fg.num_levels, fg.neighbors_count, fg.level0_neighbors_count, fg.entry, fg.n, fg.node_row, fg.adj, fg.child)
    ix.set_graph_metadata(mg.md_bits, mg.md_mags, mg.node_id, mg.node_md, mg.pseudo_entry)
    return ix


def assert_oracle(ix, mg, raw, q, filters, k, ef, shortlist=64):
    """GPU search == oracle search: arrays for every query, evaluation / pop counts for the error-free ones"""
    got = ix.batch_search_filtered(q, filters, k, ef_search=ef, shortlist_size=shortlist)
    want = pymeta.search_batch_md(mg, raw, q, filters, k, ef_search=ef, shortlist_size=shortlist)
    assert np.array_equal(got[3], want[3])
    assert np.array_equal(got[2], want[2])
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(bits(got[1]), bits(want[1]))
    sel = np.flatnonzero(want[3] == 0)
    sub = [filters[i] for i in sel]
    e0 = ix.hnsw_counters()
    ix.batch_search_filtered(q[sel], sub, k, ef_search=ef, shortlist_size=shortlist)
    e1 = ix.hnsw_counters()
    w = pymeta.search_batch_md(mg, raw, q[sel], sub, k, ef_search=ef, shortlist_size=shortlist)
    assert (e1[0] - e0[0], e1[1] - e0[1]) == (w[4], w[5])
    return want


@pytest.mark.parametrize("st,metric,dim", [(ST.HalfPrecisionFP, MK.Cosine, 768), (ST.HalfPrecisionFP, MK.DotProduct, 769),
                                           (ST.BFloat16, MK.Cosine, 769), (ST.UnsignedByte, MK.Cosine, 40),
                                           (ST.SubByte2, MK.DotProduct, 40), (ST.FullPrecisionFP, MK.Cosine, 769)])
@pytest.mark.parametrize("ef,shortlist", [(1, 64), (8, 64), (40, 5), (128, 64)])
def test_warp_md_kernel_matches_oracle(st, metric, dim, ef, shortlist):
    vecs, mg = mdgraph.build(n=500, dim=dim, md_dims=7, levels=3, nb=8, nb0=16, storage_type=int(st), metric=int(metric), seed=31)
    q, filters = with_edge_filters(*mdgraph.make_queries(vecs, mg, 48, seed=3), mg.md_dims)
    ix = md_index(vecs, mg, st, metric)
    want = assert_oracle(ix, mg, vecs, q, filters, 10, ef, shortlist)
    assert (want[3] == 0).sum() > 30
    if ef >= 8:                                                         # ef 1 pops only the roots' children: often no row is left
        assert (want[2] > 0).sum() > 20
    if metric == MK.Cosine:
        assert want[3][1] == 4 and want[3][2] == 4                     # Some([]) and the all-zero filter
    ix.close()


def test_more_queries_than_one_chunk():
    vecs, mg = mdgraph.build(n=600, dim=24, md_dims=6, storage_type=int(ST.HalfPrecisionFP), metric=int(MK.Cosine), seed=8)
    q, filters = mdgraph.make_queries(vecs, mg, 2100, seed=4)
    ix = md_index(vecs, mg, ST.HalfPrecisionFP, MK.Cosine)
    assert_oracle(ix, mg, vecs, q, filters, 5, 16)
    ix.close()


def exported(ix, md_bits, md_mags, st, metric):
    g = ix.read_graph()
    ids, mds = ix.read_graph_metadata()
    codes, mags = ix.read_codes(0, ix.size)
    fg = pyhnsw.FlatGraph(int(metric), int(st), ix.dim, codes, mags, g["root_row"], g["num_levels"], g["neighbors_count"],
                          g["level0_neighbors_count"], g["entry"], g["node_row"], g["adj"], g["child"])
    return pymeta.MdGraph(fg, md_bits, md_mags, ids, mds, 1)


def test_graphs_built_grown_shrunk_and_loaded(tmp_path):
    st, metric, dim, levels, nb, nb0, efc = ST.HalfPrecisionFP, MK.Cosine, 32, 4, 8, 16, 32
    n, n_a = 500, 300
    gp = grown_population(n, n_a, dim, levels, seed=23)
    vecs = gp["vecs"]
    raw = np.concatenate([vecs[:n_a], np.zeros((2, dim), np.float32), vecs[n_a:]])
    rng = np.random.default_rng(2)
    q = (vecs[rng.integers(0, n, 64)] + 0.03 * rng.normal(size=(64, dim))).astype(np.float32).clip(-0.999, 0.999)
    pats = np.concatenate([gp["md_bits"][2:], gp["new_bits"]])
    filters = [None if i % 3 == 0 else [pats[j % len(pats)].astype(np.int8) for j in range(i, i + 1 + i % 3)] for i in range(64)]
    ix, failed = build_a(gp, st, metric, levels, nb, nb0, efc, 64)
    assert not failed.any()
    assert_oracle(ix, exported(ix, gp["md_bits"], gp["md_mags"], st, metric), raw, q, filters, 10, 40)
    assert not insert_b(ix, gp, efc, 64, 1).any()
    md_bits, md_mags = full_table(gp)
    assert_oracle(ix, exported(ix, md_bits, md_mags, st, metric), raw, q, filters, 10, 40)
    dead = np.concatenate([rng.choice(n_a, 20, replace=False), n_a + 2 + rng.choice(n - n_a, 10, replace=False)]).astype(np.uint32)
    ix.delete_rows_replicas(dead, 64, 64)
    assert_oracle(ix, exported(ix, md_bits, md_mags, st, metric), raw, q, filters, 10, 40)
    ix.close()
    src, lx, hf = cold_start(gp, st, metric, levels, nb, nb0, efc, str(tmp_path / "idx"))
    lx.set_graph_slot_scores(hf.slot_scores, hf.slot_tags)
    assert_oracle(lx, exported(lx, hf.md_bits, hf.md_mags, st, metric), raw, q, filters, 10, 40)
    hf.close(); lx.close(); src.close()


@pytest.mark.parametrize("st,metric,dim", [(ST.HalfPrecisionFP, MK.Cosine, 768), (ST.UnsignedByte, MK.DotProduct, 40)])
def test_edge_filters_and_the_plain_entry_point_match_oracle(st, metric, dim):
    vecs, mg = mdgraph.build(n=500, dim=dim, md_dims=7, levels=3, storage_type=int(st), metric=int(metric), seed=12)
    q, filters = with_edge_filters(*mdgraph.make_queries(vecs, mg, 64, seed=6), mg.md_dims)
    ix = md_index(vecs, mg, st, metric)
    assert_oracle(ix, mg, vecs, q, filters, 10, 64)
    # the plain entry point on the same graph: every query unfiltered, deduplicated by replica id (root and pseudo nodes
    # dropped) and re-ranked on the base vectors
    got = ix.batch_search(q, 10, cdb.SearchMode.HNSW, ef_search=64, shortlist_size=64)
    want = pymeta.search_batch_md(mg, vecs, q, [None] * q.shape[0], 10, ef_search=64, shortlist_size=64)
    assert np.array_equal(got[3], want[3]) and np.array_equal(got[2], want[2])
    assert np.array_equal(got[0], want[0]) and np.array_equal(bits(got[1]), bits(want[1]))
    assert (want[2] > 0).sum() > 32
    ix.close()


class DeviceBatch:
    """queries and CSR filters on the GPU, outputs allocated there"""

    def __init__(self, ix, q, filters, k, extra_rows=0, has=True):
        offs, dims, hasf = ix.pack_filters(filters)
        self.n_rows = dims.shape[0]
        pad = np.full((extra_rows, ix.md_dims), 1, np.int8)
        self.q = torch.from_numpy(np.ascontiguousarray(q, np.float32)).cuda()
        self.offs = torch.from_numpy(offs.view(np.int32)).cuda()
        self.dims = torch.from_numpy(np.concatenate([dims, pad]) if dims.size + pad.size else np.zeros((1, ix.md_dims), np.int8)).cuda()
        self.has = torch.from_numpy(hasf).cuda() if has else None
        b = q.shape[0]
        self.ids = torch.zeros((b, k), dtype=torch.int32, device="cuda")
        self.scores = torch.zeros((b, k), dtype=torch.float32, device="cuda")
        self.counts = torch.zeros(b, dtype=torch.int32, device="cuda")
        self.err = torch.zeros(b, dtype=torch.uint8, device="cuda")
        self.b, self.k = b, k

    def run(self, ix, stream, **kw):
        ix.batch_search_filtered_device(self.q.data_ptr(), self.b, self.k, self.offs.data_ptr(), self.dims.data_ptr(), self.n_rows,
                                        None if self.has is None else self.has.data_ptr(), self.ids.data_ptr(), self.scores.data_ptr(),
                                        self.counts.data_ptr(), self.err.data_ptr(), stream.cuda_stream, **kw)

    def result(self):
        return (self.ids.cpu().numpy().view(np.uint32), self.scores.cpu().numpy(), self.counts.cpu().numpy().view(np.uint32),
                self.err.cpu().numpy())


def assert_same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8))


def test_device_form_equals_host_form_on_caller_streams():
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    vecs, mg = mdgraph.build(n=600, dim=64, md_dims=7, levels=3, storage_type=int(st), metric=int(metric), seed=14)
    q, filters = with_edge_filters(*mdgraph.make_queries(vecs, mg, 300, seed=7), mg.md_dims)
    ix = md_index(vecs, mg, st, metric)
    k, kw = 10, dict(ef_search=48, shortlist_size=64)
    host = ix.batch_search_filtered(q, filters, k, **kw)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = DeviceBatch(ix, q, filters, k)
    b = DeviceBatch(ix, q[::-1].copy(), filters[::-1], k)
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    for _ in range(3):                                                  # two streams on one handle, enqueued interleaved
        a.run(ix, s1, **kw)
        b.run(ix, s2, **kw)
    s1.synchronize(); s2.synchronize()
    assert_same(a.result(), host)
    assert_same(b.result(), tuple(np.asarray(x)[::-1] for x in host))
    # null d_has_filter: every query unfiltered, as the host form with no filters
    c = DeviceBatch(ix, q, filters, k, has=False)
    c.run(ix, s1, **kw)
    s1.synchronize()
    assert_same(c.result(), ix.batch_search_filtered(q, [None] * q.shape[0], k, **kw))
    ix.close()


def test_bad_filter_ranges_fail_only_their_queries():
    st, metric = ST.HalfPrecisionFP, MK.Cosine
    vecs, mg = mdgraph.build(n=400, dim=32, md_dims=6, levels=3, storage_type=int(st), metric=int(metric), seed=15)
    q, _ = mdgraph.make_queries(vecs, mg, 8, seed=2)
    rows = [mg.md_bits[2 + i].astype(np.int8) for i in range(4)]
    # n_filter_rows = 4; the buffer holds 12 rows (valid-looking ones), so a missing check returns results instead of faulting
    offs = np.array([0, 1, 0, 2, 9, 3, 3, 2, 4], np.uint32)
    has = np.array([1, 1, 1, 1, 1, 1, 0, 1], np.uint8)
    bad = np.array([0, 1, 0, 1, 1, 0, 0, 0], bool)                     # 1: 1 > 0; 3: 9 > n_rows; 4: 9 > 3
    ix = md_index(vecs, mg, st, metric)
    k = 5
    dev = DeviceBatch(ix, q, [[r] for r in rows] * 2, k)                 # shapes only: offsets / has replaced below
    dev.offs = torch.from_numpy(offs.view(np.int32)).cuda()
    dev.has = torch.from_numpy(has).cuda()
    dev.dims = torch.from_numpy(np.concatenate([np.stack(rows), np.tile(np.stack(rows), (2, 1))])).cuda()
    dev.n_rows = 4
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    dev.run(ix, s, ef_search=32)
    s.synchronize()
    ids, scores, counts, err = dev.result()
    assert np.array_equal(err[bad], np.full(bad.sum(), BAD_FILTER, np.uint8))
    assert not counts[bad].any()
    good = np.flatnonzero(~bad)
    want_f = [None if not has[i] else rows[offs[i]:offs[i + 1]] for i in good]
    w = ix.batch_search_filtered(q[good], want_f, k, ef_search=32)
    assert_same((ids[good], scores[good], counts[good], err[good]), w)
    assert (err[good] & BAD_FILTER == 0).all() and counts[good].sum() > 0
    ix.close()


def test_shared_memory_limits_are_unchanged():
    # ef 4096 with f32 rows at D = 768 is accepted (same results as the oracle) ...
    st, metric = ST.FullPrecisionFP, MK.Cosine
    vecs, mg = mdgraph.build(n=300, dim=768, md_dims=6, levels=2, storage_type=int(st), metric=int(metric), seed=16)
    q, filters = mdgraph.make_queries(vecs, mg, 16, seed=1)
    ix = md_index(vecs, mg, st, metric)
    assert_oracle(ix, mg, vecs, q, filters, 10, 4096)
    ix.close()
    # ... and at D = 8192 it is refused: the warp's shared memory would be 217,664 bytes, over the 200 KB the search allows
    vecs, mg = mdgraph.build(n=40, dim=8192, md_dims=6, levels=2, storage_type=int(st), metric=int(metric), seed=17)
    ix = md_index(vecs, mg, st, metric)
    with pytest.raises(cdb.CosdataError) as e:
        ix.batch_search_filtered(vecs[:2], [None, None], 5, ef_search=4096)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    ix.close()
