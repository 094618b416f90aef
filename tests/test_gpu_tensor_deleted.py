"""Brute-force searches on shards with deleted rows through the tensor-core paths (CDB_SEARCH_TENSOR_WITH_DELETED): the f16
and s8 prefilters (deleted rows have zero shadow rows, the re-rank drops them) and the exact u8 / sub-byte wgmma (a tile
holding a deleted row takes the masked epilogue).  Every search is compared -- ids and score bits -- with the CPU oracle
over the live rows and with the same search without the flag (the exact scan), and stats() must show which path ran."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from cosdata_b200.sharding import ShardGroup, shard_range

pytestmark = pytest.mark.gpu
ST, MK, MODE = cdb.StorageType, cdb.DistanceMetricKind, cdb.SearchMode
N, DIM, NQ = 20077, 128, 40   # 78 full tiles of 256 rows and a partial one of 109


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def want_topk(corpus, live, q, k, st=None, metric=MK.Cosine):
    """oracle top-k over the live rows, ids mapped back (live is ascending, so ties still prefer the smaller id)"""
    if st is None:
        ids, scores = orc.brute_topk_f32(corpus[live], q, k)
        return live[ids], scores, np.zeros(len(q), np.uint8)
    codes, mags = orc.quantize_batch(int(st), corpus)
    qc, qm = orc.quantize_batch(int(st), q)
    rc, ids, scores, err = orc.brute_topk_codes(int(metric), int(st), corpus.shape[1], codes[live], mags[live], qc, qm, k)
    assert rc == 0
    return live[ids], scores, err


def search_both(ix, q, k, mode, want, expect_tensor=True, s8=None, **kw):
    """flag on (tensor path expected) and flag off (exact scan), both equal to `want`"""
    w_ids, w_scores, w_err = want
    st0 = ix.stats()
    ids, scores, counts, err = ix.batch_search(q, k, mode, tensor_with_deleted=True, **kw)
    st1 = ix.stats()
    ran = 1 if expect_tensor else 0
    assert st1["tensor_searches"] - st0["tensor_searches"] == ran, (st0, st1)
    assert st1["tensor_deleted_searches"] - st0["tensor_deleted_searches"] == ran, (st0, st1)
    if s8 is not None:
        assert st1["s8_searches"] - st0["s8_searches"] == (1 if s8 else 0), (st0, st1)
    assert np.array_equal(ids, w_ids), np.argwhere(ids != w_ids)[:5]
    assert np.array_equal(bits(scores), bits(w_scores))
    assert np.array_equal(err, w_err)
    ids2, scores2, counts2, err2 = ix.batch_search(q, k, mode, **kw)
    assert ix.stats()["tensor_searches"] == st1["tensor_searches"]   # without the flag the exact scan answered
    assert np.array_equal(ids2, ids) and np.array_equal(bits(scores2), bits(scores))
    assert np.array_equal(counts2, counts) and np.array_equal(err2, err)
    return ids, scores


# (name, storage type or None for BRUTE_RAW, metric, s8 form)
FORMS = [("raw_f16", None, MK.Cosine, False), ("raw_s8", None, MK.Cosine, True),
         ("u8_cos", ST.UnsignedByte, MK.Cosine, None), ("u8_dot", ST.UnsignedByte, MK.DotProduct, None),
         ("sub2_cos", ST.SubByte2, MK.Cosine, None), ("sub2_dot", ST.SubByte2, MK.DotProduct, None)]
PATTERNS = ["random10", "top3", "residues", "tiles", "last_tile"]


def make_index(st, metric, corpus, **kw):
    ix = cdb.DenseIndex(dim=corpus.shape[1], storage_type=ST.FullPrecisionFP if st is None else st, metric=metric,
                        capacity=kw.pop("capacity", corpus.shape[0]), **kw)
    ix.append(corpus)
    return ix


def dead_rows(pattern, n, top3):
    rng = np.random.default_rng(7)
    r = np.arange(n)
    if pattern == "random10":
        d = rng.choice(n, n // 10, replace=False)
    elif pattern == "top3":         # exactly the rows that set the class maxima
        d = top3.ravel()
    elif pattern == "residues":     # every row of three classes mod 64, in 40 tiles
        d = r[(r < 40 * 256) & np.isin(r % 64, [3, 17, 40])]
    elif pattern == "tiles":        # whole 256-row tiles
        d = np.concatenate([np.arange(5 * 256, 7 * 256), np.arange(30 * 256, 31 * 256)])
    else:                           # rows of the last, partial tile
        d = np.array([n - 1, n - 5, n - 60])
    return np.unique(d).astype(np.uint32)


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("form", FORMS, ids=[f[0] for f in FORMS])
def test_parity_matrix(form, pattern, monkeypatch):
    name, st, metric, s8 = form
    if s8 is not None:
        monkeypatch.setenv("CDB_TS_S8", "1" if s8 else "0")
    mode = MODE.BRUTE_RAW if st is None else MODE.BRUTE_CODES
    corpus = orc.synth_matrix(910 + len(name), N, DIM).copy()
    q = orc.synth_matrix(920, NQ, DIM)
    ix = make_index(st, metric, corpus)
    ids0, _, _, _ = ix.batch_search(q, 10, mode)
    dead = dead_rows(pattern, N, ids0[:, :3])
    assert (ix.delete_rows(dead) == 0).all()
    live = np.setdiff1d(np.arange(N), dead)
    for k in (1, 10, 64):
        want = want_topk(corpus, live, q, k, st, metric)
        ids, _ = search_both(ix, q, k, mode, want, s8=s8)
        assert not np.isin(ids, dead).any()
    ix.close()


@pytest.mark.parametrize("s8", [False, True])
def test_bound_adversary_zero_shadow_rows_score_above_every_live_row(s8, monkeypatch):
    """all-positive corpus, all-negative queries: every live cosine is < -0.5 while the deleted rows' zero shadow rows
    score 0 -- if they entered the class maxima the prefilter would drop the true top-k"""
    monkeypatch.setenv("CDB_TS_S8", "1" if s8 else "0")
    rng = np.random.default_rng(3)
    corpus = rng.uniform(0.1, 1.0, size=(N, DIM)).astype(np.float32)
    q = -rng.uniform(0.1, 1.0, size=(NQ, DIM)).astype(np.float32)
    ix = make_index(None, MK.Cosine, corpus)
    dead = np.unique(np.concatenate([np.arange(64) + 256 * t for t in (2, 11, 50)] + [rng.choice(N, 500, replace=False)]))
    assert (ix.delete_rows(dead.astype(np.uint32)) == 0).all()
    live = np.setdiff1d(np.arange(N), dead)
    for k in (1, 10, 64):
        ids, scores = search_both(ix, q, k, MODE.BRUTE_RAW, want_topk(corpus, live, q, k), s8=s8)
        assert not np.isin(ids, dead).any() and (scores < -0.5).all()
    ix.close()


def test_deleted_odd_rows_are_never_returned():
    corpus = orc.synth_matrix(930, N, DIM).copy()
    q = orc.synth_matrix(931, NQ, DIM)
    corpus[100, 5] = np.inf      # degenerate rows that ride on every candidate list
    corpus[7000, :] = np.nan
    corpus[9000, :] = 1e20       # norm overflows
    ix = make_index(None, MK.Cosine, corpus)
    assert ix.stats()["odd_rows"] == 3
    dead = np.array([100, 7000, 9000, 12345], np.uint32)
    assert (ix.delete_rows(dead) == 0).all()
    live = np.setdiff1d(np.arange(N), dead)
    for k in (1, 10, 64):
        ids, _ = search_both(ix, q, k, MODE.BRUTE_RAW, want_topk(corpus, live, q, k))
        assert not np.isin(ids, dead).any()
    ix.close()


def test_deleted_zero_magnitude_row_raises_no_error_on_the_u8_cosine_path():
    corpus = orc.synth_matrix(940, N, DIM).copy()
    corpus[321] = -1.0           # all-zero u8 codes: magnitude 0
    q = orc.synth_matrix(941, NQ, DIM)
    ix = make_index(ST.UnsignedByte, MK.Cosine, corpus)
    _, _, _, err = ix.batch_search(q, 10, MODE.BRUTE_CODES)
    w_err = want_topk(corpus, np.arange(N), q, 10, ST.UnsignedByte, MK.Cosine)[2]
    assert w_err.any() and np.array_equal(err, w_err)   # while live, the zero-magnitude row is an Err
    assert (ix.delete_rows([321, 322]) == 0).all()
    live = np.setdiff1d(np.arange(N), [321, 322])
    want = want_topk(corpus, live, q, 10, ST.UnsignedByte, MK.Cosine)
    assert not want[2].any()
    search_both(ix, q, 10, MODE.BRUTE_CODES, want)
    ix.close()


def test_fewer_than_k_live_proper_rows_take_the_exact_scan():
    corpus = orc.synth_matrix(950, N, DIM).copy()
    q = orc.synth_matrix(951, NQ, DIM)
    ix = make_index(None, MK.Cosine, corpus)
    keep = np.random.default_rng(4).choice(N, 80, replace=False)
    dead = np.setdiff1d(np.arange(N), keep).astype(np.uint32)
    assert (ix.delete_rows(dead) == 0).all()
    live = np.sort(keep)
    search_both(ix, q, 64, MODE.BRUTE_RAW, want_topk(corpus, live, q, 64))     # 80 live rows >= 64: prefilter
    corpus[live[:20]] = 0.0
    ix.close()
    ix = make_index(None, MK.Cosine, corpus)   # 20 of them all-zero: 60 live proper rows < 64
    assert (ix.delete_rows(dead) == 0).all()
    search_both(ix, q, 64, MODE.BRUTE_RAW, want_topk(corpus, live, q, 64), expect_tensor=False)
    ix.close()


@pytest.mark.parametrize("form", [FORMS[0], FORMS[1], FORMS[2]], ids=["raw_f16", "raw_s8", "u8_cos"])
def test_delete_then_append_into_the_open_tile_and_beyond(form, monkeypatch):
    name, st, metric, s8 = form
    if s8 is not None:
        monkeypatch.setenv("CDB_TS_S8", "1" if s8 else "0")
    mode = MODE.BRUTE_RAW if st is None else MODE.BRUTE_CODES
    n0, extra = N, 600
    corpus = orc.synth_matrix(960, n0 + extra, DIM).copy()
    q = np.concatenate([orc.synth_matrix(961, NQ, DIM), corpus[[n0 - 2, n0 - 50, 4000]]])
    ix = make_index(st, metric, corpus[:n0], capacity=n0 + extra)
    dead = np.array([4000, 10001, n0 - 50, n0 - 2], np.uint32)   # two rows of the open tile
    assert (ix.delete_rows(dead) == 0).all()
    ix.append(corpus[n0:n0 + 40])        # re-quantizes the open tile
    ix.append(corpus[n0 + 40:])
    live = np.setdiff1d(np.arange(n0 + extra), dead)
    for k in (1, 10):
        ids, _ = search_both(ix, q, k, mode, want_topk(corpus, live, q, k, st, metric), s8=s8)
        assert not np.isin(ids, dead).any()
    ix.close()


@pytest.mark.parametrize("s8", [False, True])
def test_set_raw_on_a_deleted_row_keeps_it_out(s8, monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", "1" if s8 else "0")
    corpus = orc.synth_matrix(970, N, DIM).copy()
    ix = make_index(ST.UnsignedByte, MK.Cosine, corpus, keep_raw_f32=True)
    assert (ix.delete_rows([55, 777]) == 0).all()
    v = orc.synth_matrix(971, 2, DIM)
    ix.set_raw(55, v[:1])
    ix.set_raw(777, v[1:])
    corpus[55], corpus[777] = v[0], v[1]
    q = np.concatenate([v, orc.synth_matrix(972, NQ, DIM)])   # their own vectors as queries
    live = np.setdiff1d(np.arange(N), [55, 777])
    for k in (1, 10):
        ids, _ = search_both(ix, q, k, MODE.BRUTE_RAW, want_topk(corpus, live, q, k), s8=s8)
        assert not np.isin(ids, [55, 777]).any()
    ix.close()


def test_delete_through_the_graph_shares_the_bitmap():
    n, dim = N, 64
    corpus = orc.synth_matrix(980, n, dim)
    q = orc.synth_matrix(981, NQ, dim)
    ix = cdb.DenseIndex(dim=dim, storage_type=ST.UnsignedByte, metric=MK.Cosine, capacity=n + 1, keep_raw_f32=True)
    ix.append(corpus)
    ix.build_graph(4, 16, 32, 64, 64, 4096, 3)   # appends the root row
    ids0, _, _, _ = ix.batch_search(q, 10, MODE.BRUTE_CODES)
    dead = np.unique(np.concatenate([ids0[:, :3].ravel(), np.random.default_rng(6).choice(n, 1000, replace=False)])).astype(np.uint32)
    assert (ix.delete_rows(dead) != 1).all()
    assert np.array_equal(np.flatnonzero(ix.deleted_rows()), dead)
    codes, mags = ix.read_codes(0, ix.size)
    qc, qm = orc.quantize_batch(int(ST.UnsignedByte), q)
    live = np.setdiff1d(np.arange(ix.size), dead)
    rc, wi, ws, werr = orc.brute_topk_codes(int(MK.Cosine), int(ST.UnsignedByte), dim, codes[live], mags[live], qc, qm, 10)
    assert rc == 0
    search_both(ix, q, 10, MODE.BRUTE_CODES, (live[wi], ws, werr))
    ids, _, _, _ = ix.batch_search(q, 10, MODE.HNSW, ef_search=64, shortlist_size=64, tensor_with_deleted=True)
    assert not np.isin(ids, dead).any()
    ix.close()


@pytest.mark.parametrize("nq,prefilter_k", [(8, 10), (100, 10)])   # per-query fallback / whole-batch fallback
@pytest.mark.parametrize("st", [None, ST.UnsignedByte])
def test_fallbacks_with_deletes_stay_exact(st, nq, prefilter_k):
    mode = MODE.BRUTE_RAW if st is None else MODE.BRUTE_CODES
    corpus = orc.synth_matrix(990, N, DIM).copy()
    q = orc.synth_matrix(991, nq, DIM)
    ix = make_index(st, MK.Cosine, corpus)
    dead = np.random.default_rng(8).choice(N, N // 10, replace=False).astype(np.uint32)
    assert (ix.delete_rows(dead) == 0).all()
    live = np.setdiff1d(np.arange(N), dead)
    fb0 = ix.stats()["fallbacks"]
    search_both(ix, q, 10, mode, want_topk(corpus, live, q, 10, st), prefilter_k=prefilter_k)
    assert ix.stats()["fallbacks"] - fb0 == 1
    assert ix.stats()["fallback_queries"] > 0
    ix.close()


def test_sharded_with_deletes_on_one_shard():
    n, k = 40000, 10
    corpus = orc.synth_matrix(1000, n, DIM)
    q = orc.synth_matrix(1001, 33, DIM)
    g = ShardGroup.local([0, 0])
    parts = []
    for r in range(2):
        row0, cnt = shard_range(n, 2, r)
        ix = cdb.DenseIndex(dim=DIM, capacity=cnt, device=0, id_base=row0)
        ix.append(corpus[row0:row0 + cnt])
        g.attach(r, ix)
        parts.append(ix)
    row0, cnt = shard_range(n, 2, 1)
    local = np.random.default_rng(9).choice(cnt, 2000, replace=False).astype(np.uint32)
    assert (parts[1].delete_rows(local) == 0).all()
    dead = local.astype(np.int64) + row0
    live = np.setdiff1d(np.arange(n), dead)
    before = [p.stats() for p in parts]
    ids, scores, counts, err = g.search(q, k, tensor_with_deleted=True)
    after = [p.stats() for p in parts]
    assert all(a["tensor_searches"] - b["tensor_searches"] == 1 for a, b in zip(after, before))
    assert after[1]["tensor_deleted_searches"] - before[1]["tensor_deleted_searches"] == 1
    w_ids, w_scores, _ = want_topk(corpus, live, q, k)
    assert np.array_equal(ids, w_ids) and np.array_equal(bits(scores), bits(w_scores)) and not err.any()
    g.close()
    for p in parts:
        p.close()
