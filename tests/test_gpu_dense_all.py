"""Dense HNSW search without top_k (CDB_SEARCH_ALL_CANDIDATES, k=None in Python): every deduplicated candidate is re-ranked
by exact f32 cosine and the whole sorted list comes back in rows of cap = (num_levels + 1) * 100 columns.
  * plain graphs: equal to the C oracle's search_internal at k = cap (5 * cap >= cap, so it neither cuts nor truncates) --
    ids, counts, error flags and score bits -- over every storage type, uploaded graphs of 4, 12 and 31 levels and graphs of
    12 and 15 levels built on the GPU; where cap <= 1024 also bit-identical to the top-k search at k = cap;
  * replica graphs (tests/mdgraph.py), filtered and unfiltered queries: equal to the metadata oracle at k = cap, error flags
    (UNREACHABLE, CALCULATION) included, and to the top-k search at k = cap;
  * the device entry points, and the refusals: a width below cap, and k=None with a brute-force mode."""
import numpy as np
import pytest
import torch

import cosdata_b200 as cdb
from oracle import pyhnsw, pymeta
from tests import mdgraph
from tests.test_gpu_filtered_device import md_index, with_edge_filters
from tests.test_gpu_hnsw import build_both, clustered
from tests.test_gpu_hnsw_build import build_gpu, flat_from

pytestmark = pytest.mark.gpu
ST, MK, MODE = cdb.StorageType, cdb.DistanceMetricKind, cdb.SearchMode


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_equal(got, want, what=""):
    assert np.array_equal(got[3], want[3]), what
    assert np.array_equal(got[2], want[2]), what
    assert np.array_equal(got[0], want[0]), what
    assert np.array_equal(bits(got[1]), bits(want[1])), what


def queries_near(vecs, nq, seed):
    rng = np.random.default_rng(seed)
    return (vecs[rng.integers(0, len(vecs), nq)] + 0.05 * rng.normal(size=(nq, vecs.shape[1]))).astype(np.float32)


@pytest.mark.parametrize("st,metric,levels", [(ST.HalfPrecisionFP, MK.Cosine, 4), (ST.UnsignedByte, MK.Cosine, 12),
                                              (ST.SubByte1, MK.DotProduct, 4), (ST.SubByte2, MK.DotProduct, 31),
                                              (ST.SubByte3, MK.Cosine, 12), (ST.FullPrecisionFP, MK.Cosine, 31),
                                              (ST.BFloat16, MK.Cosine, 9), (ST.HalfPrecisionFP, MK.DotProduct, 31)])
def test_uploaded_graph_equals_oracle_at_k_cap(st, metric, levels):
    n, dim = 1500, 40
    vecs = clustered(n, dim, 3 + levels)
    fg, ix = build_both(vecs, st, metric, levels=levels, nb=8, nb0=16, efc=32, seed=levels)
    cap = (levels + 1) * 100
    assert ix.hnsw_out_cap() == cap
    q = queries_near(vecs, 70, levels)
    got = ix.batch_search(q, None, MODE.HNSW, ef_search=64)
    assert got[0].shape == (70, cap)
    want = pyhnsw.search_batch(fg, vecs, q, cap, ef_search=64)
    assert_equal(got, want, "top_k None vs the oracle at k = cap")
    assert (got[2] > 10).all()
    if cap <= 1024:
        assert_equal(got, ix.batch_search(q, cap, MODE.HNSW, ef_search=64), "top_k None vs the top-k search at k = cap")
    # a wider row changes nothing but the padding
    wide = ix.batch_search(q, cap + 37, MODE.HNSW, ef_search=64, all_candidates=True)
    assert_equal((wide[0][:, :cap], wide[1][:, :cap], wide[2], wide[3]), got)
    assert (wide[0][:, cap:] == cdb.INVALID_ID).all() and (bits(wide[1][:, cap:]) == 0).all()
    ix.close()


@pytest.mark.parametrize("levels", [12, 15])
def test_gpu_built_graph_equals_oracle_over_query_chunks(levels):
    n, dim = 4000, 32
    vecs = clustered(n, dim, 40 + levels)
    ix, g = build_gpu(vecs, ST.HalfPrecisionFP, MK.Cosine, levels, 8, 16, 32, 512, levels)
    fg = flat_from(ix, g, ST.HalfPrecisionFP, MK.Cosine, dim, n)
    cap = (levels + 1) * 100
    q = queries_near(vecs, 2100, levels)                                # two chunks of the single-index search
    got = ix.batch_search(q, None, MODE.HNSW, ef_search=128)
    want = pyhnsw.search_batch(fg, vecs, q, cap, ef_search=128)
    assert_equal(got, want)
    # the device form on a caller stream
    dq = torch.from_numpy(q).cuda()
    ids = torch.empty((len(q), cap), dtype=torch.int32, device="cuda")
    sc = torch.empty((len(q), cap), dtype=torch.float32, device="cuda")
    cnt = torch.empty(len(q), dtype=torch.int32, device="cuda")
    err = torch.empty(len(q), dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    ix.batch_search_device(dq.data_ptr(), len(q), cap, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), err.data_ptr(), st.cuda_stream,
                           mode=MODE.HNSW, ef_search=128, all_candidates=True)
    st.synchronize()
    assert_equal((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32), err.cpu().numpy()), want)
    ix.close()


def test_replica_graph_filtered_and_unfiltered_equal_the_metadata_oracle():
    vecs, mg = mdgraph.build(n=500, dim=40, md_dims=7, levels=5, nb=8, nb0=16, storage_type=int(ST.HalfPrecisionFP),
                             metric=int(MK.Cosine), seed=31)
    q, filters = with_edge_filters(*mdgraph.make_queries(vecs, mg, 64, seed=3), mg.md_dims)
    ix = md_index(vecs, mg, ST.HalfPrecisionFP, MK.Cosine)
    cap = 600
    got = ix.batch_search_filtered(q, filters, None, ef_search=64)
    want = pymeta.search_batch_md(mg, vecs, q, filters, cap, ef_search=64)
    assert_equal(got, want, "filtered")
    assert want[3][1] == 4 and want[3][2] == 4                          # Some([]) and the all-zero filter: UNREACHABLE
    assert (want[2] > 10).sum() > 40
    assert_equal(got, ix.batch_search_filtered(q, filters, cap, ef_search=64), "filtered vs k = cap")
    # unfiltered: the filtered entry without filters and the plain entry
    none = [None] * len(q)
    want = pymeta.search_batch_md(mg, vecs, q, none, cap, ef_search=64)
    assert_equal(ix.batch_search_filtered(q, none, None, ef_search=64), want, "unfiltered, filtered entry")
    assert_equal(ix.batch_search(q, None, MODE.HNSW, ef_search=64), want, "unfiltered, plain entry")
    ix.close()


def test_replica_graph_calculation_errors_and_device_form():
    vecs, mg = mdgraph.build(n=400, dim=24, md_dims=6, levels=3, nb=8, nb0=16, storage_type=int(ST.HalfPrecisionFP),
                             metric=int(MK.Cosine), seed=8)
    q, filters = mdgraph.make_queries(vecs, mg, 48, seed=4)
    q[4] = 0.0                                                          # unfiltered, |q| = 0: a zero cosine denominator
    ix = md_index(vecs, mg, ST.HalfPrecisionFP, MK.Cosine)
    cap = 400
    want = pymeta.search_batch_md(mg, vecs, q, filters, cap, ef_search=32)
    got = ix.batch_search_filtered(q, filters, None, ef_search=32)
    assert_equal(got, want)
    assert want[3][4] == 1                                             # CALCULATION
    offs, dims, has = ix.pack_filters(filters)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in (("q", q), ("o", offs.view(np.int32)), ("d", dims), ("h", has))}
    ids = torch.empty((len(q), cap), dtype=torch.int32, device="cuda")
    sc = torch.empty((len(q), cap), dtype=torch.float32, device="cuda")
    cnt = torch.empty(len(q), dtype=torch.int32, device="cuda")
    err = torch.empty(len(q), dtype=torch.uint8, device="cuda")
    ix.batch_search_filtered_device(t["q"].data_ptr(), len(q), cap, t["o"].data_ptr(), t["d"].data_ptr(), dims.shape[0],
                                    t["h"].data_ptr(), ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), err.data_ptr(), None,
                                    ef_search=32, all_candidates=True)
    torch.cuda.synchronize()
    assert_equal((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32), err.cpu().numpy()), want)
    ix.close()


def test_refusals():
    n, dim = 600, 16
    vecs = clustered(n, dim, 9)
    fg, ix = build_both(vecs, ST.HalfPrecisionFP, MK.Cosine, levels=3, nb=8, nb0=16, efc=16, seed=2)
    q = queries_near(vecs, 4, 1)
    with pytest.raises(cdb.CosdataError) as e:
        ix.batch_search(q, 399, MODE.HNSW, all_candidates=True)         # cap 400
    assert e.value.status == cdb.Status.INVALID_PARAMS
    for mode in (MODE.BRUTE_RAW, MODE.BRUTE_CODES):
        with pytest.raises(cdb.CosdataError) as e:
            ix.batch_search(q, None, mode)
        assert e.value.status == cdb.Status.INVALID_PARAMS
    for k in (0, 1025):                                                 # without the flag: unchanged
        with pytest.raises(cdb.CosdataError) as e:
            ix.batch_search(q, k, MODE.HNSW)
        assert e.value.status == cdb.Status.INVALID_PARAMS
    assert ix.batch_search(q, 400, MODE.HNSW, all_candidates=True)[2].max() > 0
    ix.close()
