"""wgmma u8 path (tensor_scan_u8.cu): exact integer scoring of u8 / sub-byte codes must equal the
CPU oracle bit for bit -- scores, ids (ties broken by smaller id: quantized scores tie often), error flags."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def run_case(st, metric, n, dim, nq, k=10, zero_row=None, expect_fallback=None, expect_tensor=True, **kw):
    corpus = orc.synth_matrix(4000 + int(st) + dim, n, dim).copy()
    if zero_row is not None:
        corpus[zero_row] = 0.0
    q = orc.synth_matrix(4100 + int(st) + nq, nq, dim)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n)
    ix.append(corpus)
    ids, scores, counts, err = ix.batch_search(q, k, cdb.SearchMode.BRUTE_CODES, **kw)
    stt = ix.stats()
    assert stt["tensor_searches"] == (1 if expect_tensor else 0), "u8 tensor-core path: ran / did not run against expectation"
    if expect_fallback is not None:
        assert (stt["fallbacks"] == 1) == expect_fallback, stt
    codes, mags = orc.quantize_batch(int(st), corpus)
    qc, qm = orc.quantize_batch(int(st), q)
    rc, want_ids, want_scores, want_err = orc.brute_topk_codes(int(metric), int(st), dim, codes, mags, qc, qm, k)
    assert rc == 0
    assert np.array_equal(err, want_err)
    assert np.array_equal(ids, want_ids)
    assert np.array_equal(bits(scores), bits(want_scores))
    # the generic exact scan agrees as well
    ids2, scores2, _, err2 = ix.batch_search(q, k, cdb.SearchMode.BRUTE_CODES, exact_only=True)
    assert np.array_equal(ids2, ids) and np.array_equal(bits(scores2), bits(scores)) and np.array_equal(err2, err)
    ix.close()


@pytest.mark.parametrize("metric", [MK.Cosine, MK.DotProduct])
@pytest.mark.parametrize("st,dim", [(ST.UnsignedByte, 768), (ST.UnsignedByte, 100), (ST.SubByte2, 1024), (ST.SubByte2, 72),
                                     (ST.SubByte1, 1024), (ST.SubByte3, 256)])
def test_i8_tensor_scan_matches_oracle(st, dim, metric):
    run_case(st, metric, 20000, dim, 5)


@pytest.mark.parametrize("nq", [1, 130])
def test_i8_tensor_scan_batch_shapes(nq):
    run_case(ST.SubByte2, MK.DotProduct, 33000, 1024, nq, expect_fallback=False)       # config C4 shape at reduced N
    run_case(ST.UnsignedByte, MK.Cosine, 33000, 768, nq, expect_fallback=False)        # the reference's default storage


def test_i8_cosine_zero_norm_row_sets_error_flags():
    run_case(ST.SubByte2, MK.Cosine, 20000, 256, 7, zero_row=1234)
    run_case(ST.UnsignedByte, MK.Cosine, 20000, 64, 7, zero_row=17)


@pytest.mark.parametrize("k", [1, 13, 29, 64, 100])
def test_i8_k_sweep(k):
    # k <= 64: class-maximum bound with 16 / 32 / 64 classes; above: the exact SIMT scan answers
    run_case(ST.SubByte2, MK.DotProduct, 20000, 512, 9, k=k, expect_tensor=k <= 64)


def test_i8_many_ties_and_low_selectivity():
    # binary codes, tiny dimension: scores take few distinct values, nearly every row ties with the k-th best -> the filter
    # must keep ALL ties (ids decide) and the lists get long
    run_case(ST.SubByte1, MK.DotProduct, 30000, 16, 40, k=10)
    run_case(ST.SubByte1, MK.Cosine, 30000, 24, 40, k=10)


def test_i8_overflow_falls_back():
    run_case(ST.SubByte2, MK.DotProduct, 20000, 128, 6, expect_fallback=True, prefilter_k=8)
