"""Refusals of dense top_k None and of the filtered sharded entries that need a device to reach:
  * a group slot without a shard is refused with CDB_INVALID_PARAMS by every dense sharded entry, flag or not (the device
    forms of a per-rank group included), before any shard is read;
  * the filtered sharded search refuses a width that is not a multiple of the world size or below a shard's cap, and the
    per-rank device form a width below its shard's cap;
  * a dimension too large for the re-rank of every candidate is refused before any device work, while the same index with
    fewer levels searches;
  * ShardGroup.all_width needs an explicit width on a per-rank group of more than one rank."""
import ctypes as C

import numpy as np
import pytest
import torch

import cosdata_b200 as cdb
from cosdata_b200 import _lib
from cosdata_b200.sharding import ShardGroup
from tests.test_gpu_hnsw import build_both, clustered
from tests.test_gpu_sharded_filtered import group_of, md_shard

pytestmark = pytest.mark.gpu
ST, MK, MODE = cdb.StorageType, cdb.DistanceMetricKind, cdb.SearchMode
INV = cdb.Status.INVALID_PARAMS
ALL = 2


def last_error():
    return _lib.load().cdb_last_error_string().decode()


def test_unattached_slots_are_refused_by_every_dense_sharded_entry():
    L = _lib.load()
    nq, dim, k = 4, 24, 10
    q = torch.zeros((nq, dim), dtype=torch.float32, device="cuda")
    ids = torch.zeros((nq, 800), dtype=torch.int32, device="cuda")
    sc = torch.zeros((nq, 800), dtype=torch.float32, device="cuda")
    offs = torch.zeros(nq + 1, dtype=torch.int32, device="cuda")
    h_q = np.zeros((nq, dim), np.float32)
    h_ids = np.zeros((nq, 800), np.uint32)
    h_sc = np.zeros((nq, 800), np.float32)
    h_offs = np.zeros(nq + 1, np.uint32)
    for flags, width in ((0, k), (ALL, 800)):
        p = _lib.SearchParams(width, int(MODE.HNSW), 64, 64, 0, 0, flags, 0)
        rank = ShardGroup.rank(None, 1, 0, 0)                            # per-rank group, nothing attached
        assert L.cdb_search_batch_sharded_device(rank._h, q.data_ptr(), nq, C.byref(p), ids.data_ptr(), sc.data_ptr(), None, None,
                                                 None) == INV
        assert last_error() == "a group slot has no shard attached"
        assert L.cdb_search_batch_filtered_sharded_device(rank._h, q.data_ptr(), nq, C.byref(p), offs.data_ptr(), None, 0, None,
                                                          ids.data_ptr(), sc.data_ptr(), None, None, None) == INV
        assert last_error() == "a group slot has no shard attached"
        rank.close()
        local = ShardGroup.local([0, 0])
        local.attach(0, md_shard(0, seed=3)[2])                          # slot 1 stays empty
        assert L.cdb_search_batch_sharded(local._h, h_q.ctypes.data, nq, C.byref(p), h_ids.ctypes.data, h_sc.ctypes.data, None,
                                          None) == INV
        assert last_error() == "a group slot has no shard attached"
        assert L.cdb_search_batch_filtered_sharded(local._h, h_q.ctypes.data, nq, C.byref(p), h_offs.ctypes.data, None, None,
                                                   h_ids.ctypes.data, h_sc.ctypes.data, None, None) == INV
        assert last_error() == "a group slot has no shard attached"
        local.close()
    torch.cuda.synchronize()


def test_filtered_sharded_width_refusals():
    shards = [md_shard(s, seed=61 + s)[2] for s in range(2)]               # caps 400 and 400
    g = group_of(shards)
    q = np.zeros((3, 24), np.float32) + 0.1
    filters = [None, [np.ones(6, np.int8)], None]
    for width, what in ((801, "a multiple of the world size"), (798, "<= k / world")):
        with pytest.raises(cdb.CosdataError) as e:
            g.search_filtered(q, filters, None, width=width)
        assert e.value.status == INV and what in str(e.value), str(e.value)
    got = g.search_filtered(q, filters, None, width=800)
    assert got[0].shape == (3, 800) and got[2].max() > 0
    g.close()
    # per-rank group of world 1, device form: a width below the shard's cap
    vecs, mg, ix = md_shard(0, seed=71)
    r = ShardGroup.rank(None, 1, 0, 0)
    r.attach(0, ix)
    offs, dims, has = ix.pack_filters(filters)
    t = {n: torch.from_numpy(np.ascontiguousarray(v)).cuda() for n, v in (("q", q), ("o", offs.view(np.int32)), ("d", dims), ("h", has))}
    out = torch.zeros((3, 400), dtype=torch.int32, device="cuda")
    sc = torch.zeros((3, 400), dtype=torch.float32, device="cuda")
    with pytest.raises(cdb.CosdataError) as e:
        r.search_filtered_device(t["q"].data_ptr(), 3, 399, t["o"].data_ptr(), t["d"].data_ptr(), dims.shape[0], t["h"].data_ptr(),
                                 out.data_ptr(), sc.data_ptr(), all_candidates=True)
    assert e.value.status == INV and "<= k / world" in str(e.value)
    r.search_filtered_device(t["q"].data_ptr(), 3, 400, t["o"].data_ptr(), t["d"].data_ptr(), dims.shape[0], t["h"].data_ptr(),
                             out.data_ptr(), sc.data_ptr(), all_candidates=True)
    torch.cuda.synchronize()
    r.close()
    for x in shards + [ix]:
        x.close()


def test_dimension_too_large_for_the_rerank_of_every_candidate_is_refused_up_front():
    dim = 43009                                                         # 4 * 43012 + 8 * 4096 > 200 KB at 31 levels (cap 3200)
    vecs = clustered(40, dim, 5)
    _, ix = build_both(vecs, ST.HalfPrecisionFP, MK.Cosine, levels=31, nb=4, nb0=8, efc=8, seed=2)
    q = vecs[:2] + np.float32(0.01)
    with pytest.raises(cdb.CosdataError) as e:
        ix.batch_search(q, None, MODE.HNSW, ef_search=8)
    assert e.value.status == INV and "dimension too large" in str(e.value), str(e.value)
    g = ShardGroup.local([0])
    g.attach(0, ix)
    with pytest.raises(cdb.CosdataError) as e:
        g.search(q, None, MODE.HNSW, ef_search=8)
    assert e.value.status == INV and "dimension too large" in str(e.value), str(e.value)
    g.close()
    ix.close()


def test_all_width_needs_an_explicit_width_on_multi_rank_groups():
    g = ShardGroup.rank(None, 1, 0, 0)
    g._ranks_elsewhere = True                                            # what ShardGroup.rank sets for world > 1
    with pytest.raises(ValueError):
        g.all_width()
    assert g.all_width(1600) == 1600
    g.close()
