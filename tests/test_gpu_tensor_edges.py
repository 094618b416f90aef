"""Tensor-core brute-force paths at their edges: an adversarial fp16 corpus, tile and batch boundaries, large dimensions,
degenerate rows and the top of the id range.  Every case compares ids and score bits with the CPU oracle and asserts
which path answered (tensor_searches / fallbacks)."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from tests import prefilter_adversary as pa

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
KS = [1, 10, 12, 13, 28, 29, 64]
CHUNK = 2048                      # queries per search chunk (search_device_locked)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tensor_chunks(nq, min_queries=4):
    """search chunks that take a tensor-core path (the f16 form needs >= 4 queries in a chunk, the u8 form one)"""
    return sum(1 for off in range(0, nq, CHUNK) if min(CHUNK, nq - off) >= min_queries)


def search_f32(ix, corpus, q, k, tensor, id_base=0, **kw):
    st0 = ix.stats()
    ids, scores, counts, err = ix.batch_search(q, k, **kw)
    st1 = ix.stats()
    want_ids, want_scores = orc.brute_topk_f32(corpus, q, k)
    assert np.array_equal(ids, want_ids + np.uint32(id_base)), "top-k ids differ from the oracle"
    assert np.array_equal(bits(scores), bits(want_scores)), "scores not bit-identical"
    assert st1["tensor_searches"] - st0["tensor_searches"] == tensor, (st0, st1)
    assert st1["fallbacks"] == st0["fallbacks"], (st0, st1)
    return ids, scores


# ------------------------------------------------------------------ adversarial fp16 corpus
@pytest.mark.parametrize("n", [16384, 16385, 40003])
@pytest.mark.parametrize("dim", [32, 64, 128, 768])
def test_adversarial_corpus(dim, n):
    x, q130, nb = pa.corpus(n, dim, 130, seed=dim + n)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    for nq in (4, 130):
        q = q130[:nq]
        for k in KS:
            ids, _ = search_f32(ix, x, q, k, tensor=1)
            if dim >= 64:
                # the answer is each query's own targets: the rows the fp16 errors push below the decoys (at D = 32
                # every block shares the same coordinates, and another block's rows can come closer)
                blk = (np.arange(nq) % nb) * pa.BLOCK
                assert ((ids >= blk[:, None]) & (ids < blk[:, None] + pa.NT)).all()
    ix.close()


# ------------------------------------------------------------------ tile and batch edges
@pytest.mark.parametrize("n", [16383, 16384, 16385, 16639])
def test_f16_row_count_edges(n):
    dim = 64
    x = orc.synth_matrix(5000 + n, n, dim)
    q = orc.synth_matrix(5001, 4, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    search_f32(ix, x, q, 10, tensor=int(n >= 16384))
    ix.close()


def test_f16_batch_edges():
    n, dim = 16385, 32
    sms = sm_count()
    x = orc.synth_matrix(5100, n, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    for nq in (3, 4, 127, 128, 129, 2048, sms * 128, sms * 128 + 1):
        q = orc.synth_matrix(5101, nq, dim)
        search_f32(ix, x, q, 10, tensor=tensor_chunks(nq))
    ix.close()


def u8_case(ix, st, metric, dim, codes, mags, q, k, tensor):
    qc, qm = orc.quantize_batch(int(st), q)
    st0 = ix.stats()
    ids, scores, counts, err = ix.batch_search(q, k, cdb.SearchMode.BRUTE_CODES)
    st1 = ix.stats()
    rc, want_ids, want_scores, want_err = orc.brute_topk_codes(int(metric), int(st), dim, codes, mags, qc, qm, k)
    assert rc == 0
    assert np.array_equal(err, want_err)
    assert np.array_equal(ids, want_ids), "top-k ids differ from the oracle"
    assert np.array_equal(bits(scores), bits(want_scores)), "scores not bit-identical"
    assert st1["tensor_searches"] - st0["tensor_searches"] == tensor, (st0, st1)
    assert st1["fallbacks"] == st0["fallbacks"], (st0, st1)


@pytest.mark.parametrize("metric", [MK.Cosine, MK.DotProduct])
@pytest.mark.parametrize("st", [ST.UnsignedByte, ST.SubByte2])
def test_u8_tile_and_batch_edges(st, metric):
    dim = 96
    for n in (16383, 16384, 16639):
        x = orc.synth_matrix(5200 + n, n, dim)
        codes, mags = orc.quantize_batch(int(st), x)
        ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n)
        ix.append(x)
        nqs = (3, 4, 129, 2048) if n == 16639 else (4,)
        for nq in nqs:
            q = orc.synth_matrix(5201 + nq, nq, dim)
            u8_case(ix, st, metric, dim, codes, mags, q, 10, tensor_chunks(nq, 1) if n >= 16384 else 0)
        ix.close()


# ------------------------------------------------------------------ dimensions
@pytest.mark.parametrize("dim", [8, 63, 65, 127, 129, 2048, 4096, 12287, 12288, 16384])
def test_f16_dimensions(dim):
    n, nq, k = 16384, 4, 10
    x = orc.synth_matrix(5300 + dim, n, dim)
    q = orc.synth_matrix(5301 + dim, nq, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    if dim >= 2048:
        ix.append_synthetic(5300 + dim, n)
    else:
        ix.append(x)
    search_f32(ix, x, q, k, tensor=1)
    ix.close()


@pytest.mark.parametrize("dim", [32896, 32897, 33025, 33026])
def test_u8_dimensions_near_the_s32_limit(dim):
    # all-255 and near-255 rows: the s32 accumulator reaches 255^2 * D, which stops being a finite float bit pattern at
    # D = 32897 and wraps at D = 33026.  Above 255^2 * D <= 0x7F7FFFFF the exact scan must answer.
    n, nq, k = 16384, 4, 10
    rng = np.random.default_rng(dim)
    codes = np.full((n, dim), 255, np.uint8)
    lowered = rng.integers(0, 400, n)
    lowered[[5, 9000, 16383]] = 0                         # three rows of all 255
    for i in np.nonzero(lowered)[0]:
        codes[i, rng.choice(dim, lowered[i], replace=False)] = 254
    mags = np.full(n, 255.0 * np.sqrt(dim), np.float32)
    q = np.ones((nq, dim), np.float32)
    q[1:, :7] = 0.99
    tensor = int(255 * 255 * dim <= 0x7F7FFFFF)
    for metric in (MK.DotProduct, MK.Cosine):
        ix = cdb.DenseIndex(dim=dim, storage_type=ST.UnsignedByte, metric=metric, capacity=n)
        ix.append_codes(codes, mags)
        u8_case(ix, ST.UnsignedByte, metric, dim, codes, mags, q, k, tensor)
        ix.close()


# ------------------------------------------------------------------ degenerate rows
def negative_corpus(n, dim, odd):
    corpus = (np.abs(orc.synth_matrix(5400, n, dim)) * 0.9 + 0.1).astype(np.float32)      # all positive
    corpus[odd] = -1e-25                    # norm underflows to 0, dp with a negative query > 0 -> +inf
    q = (-(np.abs(orc.synth_matrix(5401, 8, dim)) * 0.9 + 0.1)).astype(np.float32)       # all negative
    return corpus, q


def test_64_odd_rows_fill_the_top_64_without_duplicates():
    # every real cosine is negative, so the threshold is <= 0 and the odd rows (zero shadow, a = 0) are emitted again on
    # top of their pre-seeded copies: the re-rank must drop the duplicates
    n, dim = 20000, 64
    odd = np.sort(np.random.default_rng(1).choice(n, 64, replace=False))
    corpus, q = negative_corpus(n, dim, odd)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(corpus)
    assert ix.stats()["odd_rows"] == 64
    ids, scores = search_f32(ix, corpus, q, 64, tensor=1)
    assert (ids == odd[None, :]).all() and np.isposinf(scores).all()
    ix.close()


def test_65_odd_rows_disable_the_prefilter():
    n, dim = 20000, 64
    odd = np.sort(np.random.default_rng(2).choice(n, 65, replace=False))
    corpus, q = negative_corpus(n, dim, odd)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(corpus)
    assert ix.stats()["odd_rows"] == 65
    search_f32(ix, corpus, q, 64, tensor=0)
    ix.close()


def test_odd_rows_over_several_appends():
    n, dim = 30000, 64
    odd = np.array([3, 4000, 9999, 10000, 17000, 25000, 29999])
    corpus, q = negative_corpus(n, dim, odd)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    for a, b in ((0, 10000), (10000, 17001), (17001, n)):
        ix.append(corpus[a:b])
    assert ix.stats()["odd_rows"] == len(odd)
    for k in (5, 10):
        search_f32(ix, corpus, q, k, tensor=1)
    ix.close()


def test_set_raw_twice_counts_degenerate_rows_once():
    n, dim = 20000, 96
    corpus = orc.synth_matrix(5500, n, dim).copy()
    corpus[np.arange(40) * 311 + 7] = 1e-25          # 40 odd rows
    corpus[[11, 12000]] = 0.0                        # 2 all-zero rows
    codes, mags = orc.quantize_batch(int(ST.UnsignedByte), corpus)
    q = orc.synth_matrix(5501, 8, dim).copy()
    q[0] = np.abs(q[0]) + 0.1
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.UnsignedByte, capacity=n, keep_raw_f32=True)
    ix.append_codes(codes, mags)
    ix.set_raw(0, corpus)
    first = ix.stats()
    assert first["odd_rows"] == 40 and first["zero_rows"] == 2
    want = search_f32(ix, corpus, q, 10, tensor=1)
    ix.set_raw(0, corpus)
    ix.set_raw(5000, corpus[5000:9000])
    again = ix.stats()
    assert again["odd_rows"] == 40 and again["zero_rows"] == 2
    got = search_f32(ix, corpus, q, 10, tensor=1)
    assert np.array_equal(got[0], want[0]) and np.array_equal(bits(got[1]), bits(want[1]))
    ix.close()


# ------------------------------------------------------------------ top of the id range
def test_last_id_below_invalid_is_returned():
    n, dim = 16384, 64
    id_base = 0xFFFFFFFF - n                         # last row: id 0xFFFFFFFE
    x = orc.synth_matrix(5600, n, dim)
    q = x[[n - 1, 0, n - 2, 77]].copy()              # query 0 is the last row itself
    ix = cdb.DenseIndex(dim=dim, capacity=n, id_base=id_base)
    ix.append(x)
    ids, _ = search_f32(ix, x, q, 10, tensor=1, id_base=id_base)
    assert ids[0, 0] == 0xFFFFFFFE
    ix.close()
    with pytest.raises(cdb.CosdataError):
        cdb.DenseIndex(dim=dim, capacity=n, id_base=id_base + 1)
