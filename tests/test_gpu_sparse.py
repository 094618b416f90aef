"""The sparse inverted index on the GPU (cdb_sparse_*) against the CPU oracle (tests/sparse_oracle.c): ids and u32-derived
scores bit-exact, re-ranked scores bit-identical, on the quirks of the reference (bits 4-8, early-termination thresholds,
zero / negative / NaN values, duplicate dims, absent dims, empty queries, ties at the k boundary), on corpora of several
row tiles appended in pieces that end mid-tile, with deletes, at batch 1 and 1024, k = 1 and 1024, through the device twin,
from 8 host threads, from an itoe store, and for the values_upper_bound sampler."""
import concurrent.futures

import numpy as np
import pytest

import cosdata_b200 as cdb
from tests import pysparse as ps
from tests.sparse_data import big_sim_rows, concat_csr, quirky_rows, slice_csr, zipf_csr

pytestmark = pytest.mark.gpu

THRS = [0.0, 0.5, 1.0, 1.7, -0.3, float("nan")]


def check(got, want):
    ids, scores, counts = got
    w_ids, w_scores, w_counts = want
    assert np.array_equal(counts, w_counts)
    assert np.array_equal(ids, w_ids)
    assert np.array_equal(np.ascontiguousarray(scores).view(np.uint32), np.ascontiguousarray(w_scores).view(np.uint32))


def run(ix, corpus, queries, k, thr=0.0, rerank=False, factor=5, bits=4, ub=1.0, deleted=None, id_base=0):
    opts = cdb.SparseSearchOptions(k, thr, rerank, factor)
    got = ix.batch_search(queries, opts)
    q = cdb.sparse_csr(queries) if isinstance(queries, list) else queries
    want = ps.search(corpus, q, k, bits=bits, ub=ub, thr=thr, rerank=rerank, factor=factor, id_base=id_base, deleted=deleted)
    check(got, want)
    return got


@pytest.mark.parametrize("bits", [4, 5, 6, 7, 8])
def test_quirks_against_the_oracle(bits):
    rows = quirky_rows(1 + bits, 3000, 40)
    rows[5] = [(7, 0.0)]                        # touched only through zero products
    rows[6] = []                                # empty row: never a candidate
    rows[7] = [(3, 0.2), (3, 0.9), (3, 0.4)]    # duplicate dims: counted thrice, the last wins the re-rank
    corpus = cdb.sparse_csr(rows)
    ub = 1.5 if bits % 2 else 1.0
    ix = cdb.SparseIndex(quantization_bits=bits, values_upper_bound=ub, capacity_rows=4000, capacity_pairs=len(corpus[1]) + 10,
                         id_base=17)
    ix.append(corpus)
    queries = quirky_rows(100 + bits, 60, 45)   # dims 40..44 are absent from the index
    queries[0] = []
    queries[1] = [(7, 0.0)]
    queries[2] = [(3, 0.5), (3, 0.5), (9, 2.0)]
    queries[3] = [(41, 1.0)]
    for thr in THRS:
        for rerank, k in ((False, 10), (True, 7), (False, 1), (True, 1000)):
            run(ix, corpus, queries, k, thr, rerank, 5, bits, ub, id_base=17)
    ix.close()


def test_empty_key_range_gives_no_candidates():
    rows = [[(1, 0.1)], [(1, 0.9)], [(2, 0.5)]]
    ix = cdb.SparseIndex(capacity_rows=8, capacity_pairs=8)
    ix.append(rows)
    ids, scores, counts = ix.batch_search([[(1, 0.05), (2, 0.01)]], cdb.SparseSearchOptions(5, 1.0))
    assert counts[0] == 0 and np.all(ids == cdb.INVALID_ID) and np.all(scores == 0)
    ix.close()


def test_ties_at_the_k_boundary_go_to_the_smaller_id():
    rows = [[(0, 0.5)] for _ in range(50)]
    corpus = cdb.sparse_csr(rows)
    ix = cdb.SparseIndex(capacity_rows=64, capacity_pairs=64, id_base=3)
    ix.append(corpus)
    ids, _, counts = run(ix, corpus, [[(0, 1.0)]], 10, id_base=3)
    assert ids[0].tolist() == list(range(3, 13))
    run(ix, corpus, [[(0, 1.0)]], 4, rerank=True, factor=3, id_base=3)
    ix.close()


def test_similarities_above_2_24_and_wrapping():
    rows, query = big_sim_rows()
    corpus = cdb.sparse_csr(rows)
    ix = cdb.SparseIndex(quantization_bits=8, values_upper_bound=1.0, capacity_rows=len(rows), capacity_pairs=len(corpus[1]))
    ix.append(corpus)
    for k, rerank in ((1, False), (5, False), (20, False), (64, False), (3, True)):
        run(ix, corpus, [query], k, 0.0, rerank, 4, bits=8, ub=1.0)
    ix.close()


def test_append_after_queued_device_searches():
    """an append rebuilds the last partial tile; searches already queued on a caller's stream see the lists as they were"""
    import ctypes as C

    import torch
    from cosdata_b200 import _lib
    corpus = zipf_csr(13, 20_000, vocab=1000, mean_pairs=40)
    queries = zipf_csr(14, 256, vocab=1000, mean_pairs=20)
    first = slice_csr(corpus, 0, 12_000)
    ix = cdb.SparseIndex(capacity_rows=20_000, capacity_pairs=len(corpus[1]), values_upper_bound=2.0)
    ix.append(first)
    opts = cdb.SparseSearchOptions(100, 0.0, True, 5)
    want = ps.search(first, queries, 100, ub=2.0, rerank=True, factor=5)
    dev = torch.device("cuda", 0)
    o, d, v = [torch.from_numpy(a.astype(t)).to(dev) for a, t in zip(queries, (np.int64, np.int32, np.float32))]
    s = torch.cuda.Stream(dev)
    outs = []
    p = opts.params()
    for _ in range(8):
        ids = torch.zeros((256, 100), dtype=torch.int32, device=dev)
        sc = torch.zeros((256, 100), dtype=torch.float32, device=dev)
        cnt = torch.zeros(256, dtype=torch.int32, device=dev)
        assert _lib.load().cdb_sparse_search_batch_device(ix.h, o.data_ptr(), d.data_ptr(), v.data_ptr(), 256, C.byref(p),
                                                          ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(), C.c_void_p(s.cuda_stream)) == 0
        outs.append((ids, sc, cnt))
    ix.append(slice_csr(corpus, 12_000, 20_000))       # same tile: rebuilt in place
    s.synchronize()
    for ids, sc, cnt in outs:
        check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), want)
    run(ix, corpus, queries, 100, 0.0, True, 5, ub=2.0)
    ix.close()


def test_failed_append_changes_nothing():
    corpus = zipf_csr(15, 5000, vocab=500, mean_pairs=10)
    ix = cdb.SparseIndex(capacity_rows=5000, capacity_pairs=len(corpus[1]))
    ix.append(slice_csr(corpus, 0, 3000))
    with pytest.raises(cdb.CosdataError):
        ix.append(concat_csr([slice_csr(corpus, 3000, 5000), slice_csr(corpus, 0, 1)]))   # one row over capacity_rows
    assert len(ix) == 3000
    queries = zipf_csr(16, 50, vocab=500, mean_pairs=8)
    run(ix, slice_csr(corpus, 0, 3000), queries, 10)
    ix.close()


def multi_tile_corpus():
    return zipf_csr(7, 100_000, vocab=3000, mean_pairs=30)


def test_tiles_appended_in_pieces_with_deletes():
    corpus = multi_tile_corpus()
    n = len(corpus[0]) - 1
    ix = cdb.SparseIndex(quantization_bits=6, values_upper_bound=3.0, capacity_rows=n, capacity_pairs=len(corpus[1]), id_base=1000)
    queries = slice_csr(zipf_csr(8, 1100, vocab=3000, mean_pairs=12), 0, 1100)
    deleted = np.zeros(n, np.uint8)
    cuts = [0, 30_001, 70_000, n]                # pieces end mid-tile (tiles hold 32768 rows)
    ix.append(slice_csr(corpus, cuts[0], cuts[1]))
    part = slice_csr(corpus, 0, cuts[1])
    dels = np.array([0, 5, 29_999, 30_000], np.uint32)
    ix.delete_embedding(dels)
    deleted[dels] = 1
    run(ix, part, slice_csr(queries, 0, 64), 10, 0.0, False, bits=6, ub=3.0, deleted=deleted[:cuts[1]], id_base=1000)
    ix.append(slice_csr(corpus, cuts[1], cuts[2]))
    ix.append(slice_csr(corpus, cuts[2], cuts[3]))
    dels2 = np.arange(40_000, 90_000, 97, dtype=np.uint32)
    ix.delete_embedding(dels2)
    deleted[dels2] = 1
    got_del, total = ix.deleted_rows()
    assert np.array_equal(got_del, deleted) and total == int(deleted.sum())
    for qs, k, rerank, thr in ((slice_csr(queries, 0, 1), 10, False, 0.0), (slice_csr(queries, 0, 1), 1024, True, 0.0),
                               (queries, 1, False, 0.3), (queries, 1024, False, 0.0), (slice_csr(queries, 0, 200), 100, True, 0.1)):
        run(ix, corpus, qs, k, thr, rerank, 5, bits=6, ub=3.0, deleted=deleted, id_base=1000)
    ix.close()


def test_device_twin_and_threads_equal_the_host_results():
    import ctypes as C

    import torch
    from cosdata_b200 import _lib
    corpus = zipf_csr(9, 40_000, vocab=2000, mean_pairs=25)
    queries = zipf_csr(10, 300, vocab=2000, mean_pairs=10)
    ix = cdb.SparseIndex(capacity_rows=40_000, capacity_pairs=len(corpus[1]), values_upper_bound=2.0)
    ix.append(corpus)
    opts = cdb.SparseSearchOptions(50, 0.0, True, 5)
    want = ix.batch_search(queries, opts)
    dev = torch.device("cuda", 0)
    o, d, v = [torch.from_numpy(a.astype(t)).to(dev) for a, t in zip(queries, (np.int64, np.int32, np.float32))]
    nq = len(queries[0]) - 1
    ids = torch.zeros((nq, 50), dtype=torch.int32, device=dev)
    scores = torch.zeros((nq, 50), dtype=torch.float32, device=dev)
    counts = torch.zeros(nq, dtype=torch.int32, device=dev)
    p = opts.params()
    s = torch.cuda.current_stream(dev)
    rc = _lib.load().cdb_sparse_search_batch_device(ix.h, o.data_ptr(), d.data_ptr(), v.data_ptr(), nq, C.byref(p), ids.data_ptr(),
                                                    scores.data_ptr(), counts.data_ptr(), C.c_void_p(s.cuda_stream))
    assert rc == 0
    s.synchronize()
    check((ids.cpu().numpy().view(np.uint32), scores.cpu().numpy(), counts.cpu().numpy().view(np.uint32)), want)
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        for got in ex.map(lambda _: ix.batch_search(queries, opts), range(16)):
            check(got, want)
    ix.close()


def test_sampling_equals_the_oracle():
    rng = np.random.default_rng(3)
    for vals in (rng.gamma(1.0, 1.5, 100_000).astype(np.float32), rng.random(5000).astype(np.float32) * 3,
                 np.array([], np.float32), np.array([np.nan, 12.0, 1.0, 0.5], np.float32)):
        for clamp in (1.0, 0.0, 50.0):
            got = cdb.sparse_sample_upper_bound(vals, clamp)
            want = ps.sample(vals, clamp)
            assert np.array_equal(got[0], want[0]) and got[1] == want[1]
    assert cdb.sparse_sample_upper_bound(np.array([], np.float32))[1] == 10.0
    a, b = rng.random(300).astype(np.float32) * 4, rng.random(500).astype(np.float32) * 2
    c1, _ = cdb.sparse_sample_upper_bound(a)
    got = cdb.sparse_sample_upper_bound(b, 1.0, c1, a.size)
    want = ps.sample(np.concatenate([a, b]), 1.0)
    assert np.array_equal(got[0], want[0]) and got[1] == want[1]


def test_append_itoe_searches_like_append(tmp_path):
    from tests.test_itoe_file import TreeMapWriter, raw_embedding
    rng = np.random.default_rng(4)
    w = TreeMapWriter()
    pairs = {}
    for i, key in enumerate(rng.choice(200_000, 400, replace=False).tolist()):
        sp = [(int(d), float(np.float32(x))) for d, x in zip(rng.integers(0, 60, 1 + i % 9), rng.random(1 + i % 9))]
        md = {"age": i, "name": "y" * (i % 5)} if i % 3 == 0 else None
        dense = [0.5] * 4 if i % 2 else None
        w.insert(1, key, raw_embedding(f"e{i}", dense, metadata=md, sparse=sp))
        pairs[key] = sp
    w.serialize(str(tmp_path))
    keys = sorted(pairs)
    a = cdb.SparseIndex(capacity_rows=1000, capacity_pairs=10_000)
    got_ids = a.append_itoe(str(tmp_path))
    assert got_ids.tolist() == keys
    b = cdb.SparseIndex(capacity_rows=1000, capacity_pairs=10_000)
    b.append([pairs[k] for k in keys])
    q = [[(int(d), 0.7)] for d in range(0, 60, 3)]
    for opts in (cdb.SparseSearchOptions(10), cdb.SparseSearchOptions(5, rerank=True)):
        check(a.batch_search(q, opts), b.batch_search(q, opts))
    a.close()
    b.close()


def test_invalid_params_are_rejected():
    ix = cdb.SparseIndex(capacity_rows=10, capacity_pairs=10)
    ix.append([[(1, 0.5)]])
    for opts in (cdb.SparseSearchOptions(0), cdb.SparseSearchOptions(1025), cdb.SparseSearchOptions(1024, rerank=True, reranking_factor=6),
                 cdb.SparseSearchOptions(10, rerank=True, reranking_factor=0)):
        with pytest.raises(cdb.CosdataError) as e:
            ix.batch_search([[(1, 1.0)]], opts)
        assert e.value.status == cdb.Status.INVALID_PARAMS
    with pytest.raises(cdb.CosdataError):
        ix.append([[(1, 0.5)]] * 10)             # capacity_rows
    with pytest.raises(cdb.CosdataError):
        ix.delete_embedding([1])                 # not appended yet
    assert len(ix) == 1
    ix.close()


def test_one_million_rows_batch_1024():
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < 8 << 30:
        pytest.skip("needs 8 GB of free device memory")
    corpus = zipf_csr(11, 1_000_000, mean_pairs=120)
    queries = zipf_csr(12, 1024, mean_pairs=40)
    ix = cdb.SparseIndex(capacity_rows=1_000_000, capacity_pairs=len(corpus[1]), values_upper_bound=3.0)
    ix.append(corpus)
    for rerank in (False, True):
        opts = cdb.SparseSearchOptions(10, 0.0, rerank, 5)
        ids, scores, counts = ix.batch_search(queries, opts)
        sample = np.arange(0, 1024, 64)
        sub = concat_csr([slice_csr(queries, int(i), int(i) + 1) for i in sample])
        want = ps.search(corpus, sub, 10, bits=4, ub=3.0, rerank=rerank, factor=5)
        check((ids[sample], scores[sample], counts[sample]), want)
    ix.close()
