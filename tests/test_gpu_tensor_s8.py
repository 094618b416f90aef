"""The s8 form of the wgmma prefilter (DESIGN.md section 5c).  Every case compares ids and score bits with exact_only and
with the CPU oracle (on a subset of the queries), and asserts which form answered (s8_searches / tensor_searches)."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from tests import prefilter_s8 as ps

pytestmark = pytest.mark.gpu
ST = cdb.StorageType
KS = [1, 10, 12, 13, 28, 29, 64]
CHUNK = 2048


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def check(ix, x, q, k, s8, tensor=None, oracle_rows=16, **kw):
    """search q; `s8` / `tensor` = expected number of chunks answered by the s8 form / by any tensor-core form"""
    chunks = (len(q) + CHUNK - 1) // CHUNK
    st0 = ix.stats()
    ids, scores, _, _ = ix.batch_search(q, k, **kw)
    st1 = ix.stats()
    ids_e, scores_e, _, _ = ix.batch_search(q, k, exact_only=True)
    assert np.array_equal(ids, ids_e), "top-k ids differ from the exact scan"
    assert np.array_equal(bits(scores), bits(scores_e)), "scores not bit-identical to the exact scan"
    if x is not None:
        want_ids, want_scores = orc.brute_topk_f32(x, q[:oracle_rows], k)
        assert np.array_equal(ids[:oracle_rows], want_ids) and np.array_equal(bits(scores[:oracle_rows]), bits(want_scores))
    assert st1["s8_searches"] - st0["s8_searches"] == s8, (st0, st1)
    assert st1["tensor_searches"] - st0["tensor_searches"] == (chunks if tensor is None else tensor), (st0, st1)
    return st1, ids


def uniform(seed, n, dim):
    return orc.synth_matrix(seed, n, dim)


@pytest.mark.parametrize("n", [16384, 256 * 65 - 1, 256 * 65 + 1])
def test_tile_edges_and_every_class_count(n):
    dim = 256
    x, q = uniform(7000 + n, n, dim), uniform(7001, 512, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    for k in KS:
        st, _ = check(ix, x, q, k, s8=1)
        assert st["fallbacks"] == 0
    ix.close()


@pytest.mark.parametrize("nq", [512, 1024, 1025, 4096])
def test_batch_sizes(nq):
    n, dim = 40000, 384
    x, q = uniform(7100, n, dim), uniform(7101, nq, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    st, _ = check(ix, x, q, 10, s8=(nq + CHUNK - 1) // CHUNK)
    assert st["fallbacks"] == 0
    cand = ix.last_candidate_counts(min(nq, CHUNK))
    assert cand.max() < 4096
    ix.close()


def test_appends_that_split_tiles_requantize_the_open_tile(monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", "1")            # the spike row's tile has E_T above the gate's limit
    n, dim = 20000, 256
    x, q = uniform(7200, n, dim).copy(), uniform(7201, 512, dim)
    x[16384 + 3] = 0.0
    x[16384 + 3, 5] = 1.0                          # raises the scale of a tile that earlier appends quantized already
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    off = 0
    for m in (100, 57, 16227, 1, 255, 3360):       # every append ends inside a tile
        ix.append(x[off:off + m])
        off += m
    assert off == n
    check(ix, x, q, 10, s8=1)
    ix.close()


def test_set_raw_twice_with_degenerate_rows():
    n, dim = 20000, 256
    corpus = uniform(7300, n, dim).copy()
    corpus[np.arange(40) * 311 + 7] = 1e-25          # 40 odd rows
    corpus[[11, 12000]] = 0.0                        # 2 all-zero rows
    codes, mags = orc.quantize_batch(int(ST.UnsignedByte), corpus)
    q = uniform(7301, 512, dim).copy()
    q[0] = np.abs(q[0]) + 0.1
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.UnsignedByte, capacity=n, keep_raw_f32=True)
    ix.append_codes(codes, mags)
    ix.set_raw(0, np.zeros_like(corpus))             # a first, wrong set of rows: every tile is quantized again below
    ix.set_raw(0, corpus)
    st, want = check(ix, corpus, q, 10, s8=1)
    assert st["odd_rows"] == 40 and st["zero_rows"] == 2 and st["fallbacks"] == 0
    ix.set_raw(5000, corpus[5000:9000])
    _, got = check(ix, corpus, q, 10, s8=1)
    assert np.array_equal(got, want)
    ix.close()


def test_zero_rows_in_every_class_with_all_negative_cosines():
    n, dim, k = 40000, 256, 10
    corpus = (np.abs(uniform(7400, n, dim)) * 0.9 + 0.1).astype(np.float32)
    zr = np.concatenate([np.arange(64) + 64 * (7 + 11 * j) for j in range(3)])
    corpus[zr] = 0.0
    q = (-(np.abs(uniform(7401, 512, dim)) * 0.9 + 0.1)).astype(np.float32)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(corpus)
    st, ids = check(ix, corpus, q, k, s8=1)
    assert st["zero_rows"] == len(zr) and st["fallbacks"] == 0 and not np.isin(ids, zr).any()
    ix.close()


@pytest.mark.parametrize("dim", [128, 256])
def test_adversarial_corpus(dim, monkeypatch):
    # the construction's residual bound is far above the gate's limit: force the s8 form
    monkeypatch.setenv("CDB_TS_S8", "1")
    n = 16384 + 300
    x, q, nb = ps.adversarial_corpus(n, dim, 512, seed=dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    for k in KS:
        _, ids = check(ix, x, q, k, s8=1)
        b0 = (np.arange(len(q)) % nb) * ps.TILE
        assert ((ids > b0[:, None]) & (ids <= b0[:, None] + 64)).all()
    ix.close()


def test_per_query_fallback_on_overflowing_clusters():
    rng = np.random.default_rng(12)
    n, dim, k = 200_000, 256, 10
    corpus = uniform(7500, n, dim).copy()
    centres = rng.normal(size=(8, dim)).astype(np.float32)
    for c in range(8):
        rows = rng.choice(n, 2000, replace=False)
        corpus[rows] = centres[c] + 1e-4 * rng.normal(size=(2000, dim)).astype(np.float32)
    q = uniform(7501, 512, dim).copy()
    q[:6] = centres[:6] + 1e-4 * rng.normal(size=(6, dim)).astype(np.float32)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(corpus)
    st, _ = check(ix, corpus, q, k, s8=1, prefilter_k=1024)
    cand = ix.last_candidate_counts(len(q))
    over = int((cand > 1024).sum())               # the cluster queries, and any other whose list overflowed
    assert (cand[:6] > 1024).all() and over < 64  # re-done one by one, not as a whole batch
    assert st["fallbacks"] == 1 and st["fallback_queries"] == over
    ix.close()


def test_outliers_above_the_limit_take_f16(monkeypatch):
    n, dim = 20000, 256
    rng = np.random.default_rng(13)
    x = rng.standard_normal((n, dim)).astype(np.float32)
    x[:, :4] *= 30                                   # a few dominant dimensions: coarse tile scales, large residuals
    q = rng.standard_normal((512, dim)).astype(np.float32)
    _, _, e = ps.quantize_corpus(x[:4096])
    assert e.max() > 1.5e-2
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    monkeypatch.delenv("CDB_TS_S8", raising=False)
    check(ix, x, q, 10, s8=0)
    monkeypatch.setenv("CDB_TS_S8", "1")             # still exact in the s8 form, only with longer candidate lists
    check(ix, x, q, 10, s8=1)
    ix.close()


def test_env_forces_either_form(monkeypatch):
    n, dim = 16384 + 77, 256
    x = uniform(7600, n, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    monkeypatch.setenv("CDB_TS_S8", "0")
    check(ix, x, uniform(7601, 1024, dim), 10, s8=0)
    monkeypatch.setenv("CDB_TS_S8", "1")
    check(ix, x, uniform(7602, 8, dim), 10, s8=1, oracle_rows=8)
    check(ix, x, uniform(7603, 8, dim), 29, s8=1, oracle_rows=8)
    monkeypatch.delenv("CDB_TS_S8")
    check(ix, x, uniform(7604, 100, dim), 10, s8=0)  # small batches keep the f16 form
    ix.close()


def test_headline_shape_10m():
    n, dim, nq = 10_000_000, 768, 1024
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append_synthetic(1, n)
    q = uniform(7700, nq, dim)
    st, _ = check(ix, None, q, 10, s8=1)
    assert st["fallbacks"] == 0
    cand = ix.last_candidate_counts(nq)
    assert cand.max() < 16384
    ix.close()
