"""Metadata-filtered dense search over a shard group (cdb_search_batch_filtered_sharded[_device]) and the sharded top_k None
search (CDB_SEARCH_ALL_CANDIDATES), on loopback groups of one device and a per-rank group of world 1.
  * filtered, k = 10: equal to merge_packed over each shard's own batch_search_filtered, error bytes OR-ed over the shards,
    on groups of 2 and 3 replica graphs with disjoint replica ids;
  * the device form on a per-rank group equals the host form, and a bad filter range gives BAD_FILTER and count 0;
  * top_k None, plain and filtered: equal to the numpy run merge (sharding.merge_runs) of each shard's top_k None results,
    with shards of different num_levels, a batch that takes more than one gather chunk, and the padding of wide rows;
  * refusals: shards with different md_dims, a shard without metadata, a width too small for a shard's cap or not a
    multiple of the world size."""
import numpy as np
import pytest
import torch

import cosdata_b200 as cdb
from cosdata_b200.sharding import INVALID_ID, ShardGroup, merge_packed, merge_runs, pack_keys
from oracle import pymeta
from tests import mdgraph
from tests.test_gpu_hnsw import clustered

pytestmark = pytest.mark.gpu
ST, MK, MODE = cdb.StorageType, cdb.DistanceMetricKind, cdb.SearchMode
ID_STRIDE = 1 << 20                      # replica ids and id ranges of shard s start at s * ID_STRIDE
BAD_FILTER = 8


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def md_shard(s, n=400, levels=3, md_dims=6, seed=1):
    """a replica graph whose replica ids are offset by s * ID_STRIDE (roots and pseudo nodes keep theirs)"""
    vecs, mg = mdgraph.build(n=n, dim=24, md_dims=md_dims, levels=levels, nb=8, nb0=16, storage_type=int(ST.HalfPrecisionFP),
                             metric=int(MK.Cosine), seed=seed)
    fg = mg.fg
    ix = cdb.DenseIndex(dim=24, storage_type=ST.HalfPrecisionFP, capacity=vecs.shape[0], keep_raw_f32=True, id_base=s * ID_STRIDE)
    ix.append(vecs)
    ix.set_graph(fg.num_levels, fg.neighbors_count, fg.level0_neighbors_count, fg.entry, fg.n, fg.node_row, fg.adj, fg.child)
    node_id = [np.where(a < pymeta.PSEUDO_ROOT_ID, a + s * ID_STRIDE, a).astype(np.uint32) for a in mg.node_id]
    ix.set_graph_metadata(mg.md_bits, mg.md_mags, node_id, mg.node_md, mg.pseudo_entry)
    return vecs, mg, ix


def plain_shard(s, n, levels, seed):
    vecs = clustered(n, 24, seed)
    ix = cdb.DenseIndex(dim=24, storage_type=ST.HalfPrecisionFP, capacity=n + 1, keep_raw_f32=True, id_base=s * ID_STRIDE)
    ix.append(vecs)
    ix.build_graph(levels, 8, 16, 32, 64, 512, seed)
    return vecs, ix


def group_of(shards):
    g = ShardGroup.local([0] * len(shards))
    for s, ix in enumerate(shards):
        g.attach(s, ix)
    return g


def padded_keys(results, w):
    """each shard's (ids, scores) -> [world, B, w] keys, zero padded"""
    out = []
    for ids, scores in results:
        keys = pack_keys(ids, scores)
        out.append(np.pad(keys, ((0, 0), (0, w - keys.shape[1]))))
    return np.stack(out)


def assert_runs(got, per_shard, width):
    """group top_k None result == merge_runs of the shards' own top_k None results, padding included"""
    ids, scores, counts, err = got
    w = max(r[0].shape[1] for r in per_shard)
    m_ids, m_scores, m_counts = merge_runs(padded_keys([r[:2] for r in per_shard], w))
    n = m_ids.shape[1]
    assert ids.shape[1] == width >= n
    assert np.array_equal(counts, m_counts)
    assert np.array_equal(ids[:, :n], m_ids)
    assert np.array_equal(bits(scores[:, :n]), bits(m_scores))
    assert (ids[:, n:] == INVALID_ID).all() and (bits(scores[:, n:]) == 0).all()
    assert np.array_equal(err, np.bitwise_or.reduce(np.stack([r[3] for r in per_shard]), axis=0))
    assert np.array_equal(counts, np.sum([r[2] for r in per_shard], axis=0))


@pytest.mark.parametrize("world", [2, 3])
def test_filtered_sharded_equals_merge_of_shard_searches(world):
    parts = [md_shard(s, seed=11 + s) for s in range(world)]
    shards = [p[2] for p in parts]
    g = group_of(shards)
    vecs, mg = parts[0][0], parts[0][1]
    q, filters = mdgraph.make_queries(vecs, mg, 90, seed=5)
    filters[1] = []                                                     # Some([]): UNREACHABLE on every shard
    k = 10
    got = g.search_filtered(q, filters, k, ef_search=48)
    per = [ix.batch_search_filtered(q, filters, k, ef_search=48) for ix in shards]
    m_ids, m_scores, m_counts = merge_packed(np.stack([pack_keys(r[0], r[1]) for r in per]), k)
    assert np.array_equal(got[0], m_ids)
    assert np.array_equal(bits(got[1]), bits(m_scores))
    assert np.array_equal(got[2], m_counts)
    assert np.array_equal(got[3], np.bitwise_or.reduce(np.stack([r[3] for r in per]), axis=0))
    assert got[3][1] & 4 and (got[2] > 0).sum() > 60
    assert (got[0][got[0] != INVALID_ID] // ID_STRIDE).max() == world - 1   # every shard contributes
    # without filters: the unfiltered search of every shard
    none = [None] * len(q)
    got = g.search_filtered(q, none, k, ef_search=48)
    per = [ix.batch_search_filtered(q, none, k, ef_search=48) for ix in shards]
    assert np.array_equal(got[0], merge_packed(np.stack([pack_keys(r[0], r[1]) for r in per]), k)[0])
    # top_k None, filtered, shards of different num_levels
    g.close()
    for ix in shards:
        ix.close()
    parts = [md_shard(s, levels=3 + s, seed=21 + s) for s in range(world)]
    shards = [p[2] for p in parts]
    g = group_of(shards)
    width = world * (3 + world) * 100
    got = g.search_filtered(q, filters, None, ef_search=48)
    assert got[0].shape == (len(q), width)
    assert_runs(got, [ix.batch_search_filtered(q, filters, None, ef_search=48) for ix in shards], width)
    g.close()
    for ix in shards:
        ix.close()


def test_sharded_top_k_none_plain_and_over_gather_chunks():
    parts = [plain_shard(0, 2500, 4, 3), plain_shard(1, 2000, 7, 4)]
    shards = [p[1] for p in parts]
    g = group_of(shards)
    rng = np.random.default_rng(7)
    q = (parts[0][0][rng.integers(0, 2500, 1450)] + 0.05 * rng.normal(size=(1450, 24))).astype(np.float32)
    per = [ix.batch_search(q, None, MODE.HNSW, ef_search=64) for ix in shards]
    got = g.search(q[:200], None, MODE.HNSW, ef_search=64)                   # width 2 * 800
    assert got[0].shape == (200, 1600)
    assert_runs(got, [tuple(a[:200] for a in r) for r in per], 1600)
    # w = 12000 columns per rank: a chunk of the 256 MB gather buffer holds 1398 queries, so 1450 take two
    got = g.search(q, 24000, MODE.HNSW, ef_search=64, all_candidates=True)
    assert_runs(got, per, 24000)
    g.close()
    for ix in shards:
        ix.close()


def test_per_rank_device_form_equals_host_form_and_flags_bad_filters():
    vecs, mg, ix = md_shard(0, seed=31)
    g = ShardGroup.rank(None, 1, 0, 0)
    g.attach(0, ix)
    q, filters = mdgraph.make_queries(vecs, mg, 40, seed=6)
    offs, dims, has = ix.pack_filters(filters)
    assert has[2] and offs[3] > offs[2]
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in (("q", q), ("o", offs.view(np.int32)), ("d", dims), ("h", has))}
    stream = torch.cuda.Stream()
    for k, kw in ((10, {}), (400, {"all_candidates": True})):
        want = g.search_filtered(q, filters, None if kw else k, ef_search=32)
        ids = torch.empty((len(q), k), dtype=torch.int32, device="cuda")
        sc = torch.empty((len(q), k), dtype=torch.float32, device="cuda")
        cnt = torch.empty(len(q), dtype=torch.int32, device="cuda")
        err = torch.empty(len(q), dtype=torch.uint8, device="cuda")
        g.search_filtered_device(t["q"].data_ptr(), len(q), k, t["o"].data_ptr(), t["d"].data_ptr(), dims.shape[0], t["h"].data_ptr(),
                                 ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), err.data_ptr(), stream.cuda_stream, ef_search=32, **kw)
        stream.synchronize()
        assert np.array_equal(ids.cpu().numpy().view(np.uint32), want[0])
        assert np.array_equal(bits(sc.cpu().numpy()), bits(want[1]))
        assert np.array_equal(cnt.cpu().numpy().view(np.uint32), want[2])
        assert np.array_equal(err.cpu().numpy(), want[3])
        assert np.array_equal(want[0], ix.batch_search_filtered(q, filters, None if kw else k, ef_search=32)[0])
    # query 2's range reversed on the device: BAD_FILTER and count 0 for it alone
    bad = offs.copy()
    bad[2], bad[3] = offs[3], offs[2]
    tb = torch.from_numpy(bad.view(np.int32)).cuda()
    ids = torch.empty((len(q), 10), dtype=torch.int32, device="cuda")
    sc = torch.empty((len(q), 10), dtype=torch.float32, device="cuda")
    cnt = torch.empty(len(q), dtype=torch.int32, device="cuda")
    err = torch.empty(len(q), dtype=torch.uint8, device="cuda")
    g.search_filtered_device(t["q"].data_ptr(), len(q), 10, tb.data_ptr(), t["d"].data_ptr(), dims.shape[0], t["h"].data_ptr(),
                             ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), err.data_ptr(), None, ef_search=32)
    torch.cuda.synchronize()
    e, c = err.cpu().numpy(), cnt.cpu().numpy()
    assert e[2] & BAD_FILTER and c[2] == 0
    assert not (e[:2] & BAD_FILTER).any() and (c[:2] > 0).any()
    g.close()
    ix.close()


def test_refusals():
    inv = cdb.Status.INVALID_PARAMS
    _, _, a = md_shard(0, md_dims=6, seed=41)
    _, _, b = md_shard(1, md_dims=7, seed=42)
    _, p = plain_shard(2, 500, 3, 43)
    q = np.zeros((3, 24), np.float32) + 0.1
    for pair, what in (((a, b), "md_dims differ"), ((a, p), "a shard without metadata")):
        g = group_of(pair)
        with pytest.raises(cdb.CosdataError) as e:
            g.search_filtered(q, [None] * 3, 10)
        assert e.value.status == inv, what
        g.close()
    g = group_of((a, p))
    assert g.search(q, 10, MODE.HNSW)[2].max() > 0                       # the unfiltered search still runs
    for width in (2 * 399, 2 * 400 + 1):                                 # caps 400 and 400; a width not a multiple of 2
        with pytest.raises(cdb.CosdataError) as e:
            g.search(q, width, MODE.HNSW, all_candidates=True)
        assert e.value.status == inv
    assert g.search(q, 800, MODE.HNSW, all_candidates=True)[2].max() > 0
    g.close()
    for ix in (a, b, p):
        ix.close()
