"""The sharded dense search (csrc/shard_group.cu) at its merge edges, on loopback groups of one device.  Every shard writes
packed keys from whichever final kernel answered its chunk (tests/sharded_plan.py names them and each case asserts
through stats() that the predicted ones ran); merge_gathered_kernel picks the best k of world * k keys per query.  Exact
modes must equal one DenseIndex over every row and the CPU oracle (ids, score bits, counts, error bytes); HNSW must equal
the merge of each shard's own search.  Also: every codes arm, ties and zero scores across shard boundaries, wide groups,
the merge's shared-memory limit, error bytes through the gather, buffer reuse, the device form and the attach checks."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from cosdata_b200.sharding import ShardGroup, merge_packed, pack_keys
from tests import sharded_plan as sp

pytestmark = pytest.mark.gpu
ST, MK, MODE = cdb.StorageType, cdb.DistanceMetricKind, cdb.SearchMode
INVALID = cdb.INVALID_ID
GAP = 1000                          # ids left free between neighbouring shards


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def layout(shards, order="asc", gap=GAP, top=False):
    """-> per slot (first corpus row, rows, id_base) and the global id of every corpus row.  Corpus rows are in id order;
    order "desc" gives slot 0 the largest ids.  top: the last row gets id 0xFFFFFFFE."""
    slots = list(range(len(shards))) if order == "asc" else list(reversed(range(len(shards))))
    lay, row0, base = [None] * len(shards), 0, 0
    for s in slots:
        lay[s] = [row0, shards[s], base]
        row0, base = row0 + shards[s], base + shards[s] + gap
    if top:
        assert shards[slots[-1]], "the shard with the largest ids needs rows"
        shift = 0xFFFFFFFE - (base - gap - 1)
        for x in lay:
            x[2] += shift
    gid = np.zeros(row0, np.uint64)
    for r0, n, b in lay:
        gid[r0:r0 + n] = b + np.arange(n)
    return [tuple(x) for x in lay], gid


def make_group(corpus, lay, **kw):
    dim = corpus.shape[1]
    g = ShardGroup.local([0] * len(lay))
    parts = []
    for s, (r0, n, base) in enumerate(lay):
        ix = cdb.DenseIndex(dim=dim, capacity=max(n, 1), id_base=base, **kw)
        if n:
            ix.append(corpus[r0:r0 + n])
        g.attach(s, ix)
        parts.append(ix)
    return g, parts


def close(g, parts, *more):
    g.close()
    for p in list(parts) + list(more):
        p.close()


def to_gid(ids, gid, live=None):
    """oracle / whole-index row numbers (rows of `live` when given) -> global ids"""
    rows = np.where(ids == INVALID, 0, ids).astype(np.int64)
    if live is not None:
        rows = live[rows]
    return np.where(ids == INVALID, INVALID, gid[rows]).astype(np.uint32)


def oracle(corpus, q, k, mode, st, metric, live=None):
    """-> (ids as corpus row numbers, scores, err) or the arm's error status"""
    c = corpus if live is None else corpus[live]
    if mode == MODE.BRUTE_RAW:
        ids, scores = orc.brute_topk_f32(c, q, k)
        err = np.zeros(len(q), np.uint8)
    else:
        codes, mags = orc.quantize_batch(int(st), c)
        qc, qm = orc.quantize_batch(int(st), q)
        rc, ids, scores, err = orc.brute_topk_codes(int(metric), int(st), c.shape[1], codes, mags, qc, qm, k)
        if rc:
            return rc
    if live is not None:
        ids = np.where(ids == INVALID, INVALID, live[np.where(ids == INVALID, 0, ids)]).astype(np.uint32)
    return ids, scores, err


def assert_exact(got, whole, want, gid, sel=None):
    """group result == whole-index result (every query) == oracle (queries `sel`, default all)"""
    ids, scores, counts, err = got
    w_ids, w_scores, w_counts, w_err = whole
    assert np.array_equal(ids, to_gid(w_ids, gid)), "group ids differ from one index over every row"
    assert np.array_equal(bits(scores), bits(w_scores)), "group scores differ from one index over every row"
    assert np.array_equal(counts, w_counts) and np.array_equal(err, w_err)
    sel = np.arange(len(ids)) if sel is None else sel
    o_ids, o_scores, o_err = want
    assert np.array_equal(ids[sel], to_gid(o_ids, gid)), "group ids differ from the oracle"
    assert np.array_equal(bits(scores[sel]), bits(o_scores)), "group scores differ from the oracle"
    assert np.array_equal(err[sel], o_err)
    assert np.array_equal(counts[sel], (o_ids != INVALID).sum(axis=1).astype(np.uint32))


def search_and_check(g, corpus, gid, q, k, mode=MODE.BRUTE_RAW, st=None, metric=MK.Cosine, whole_kw=None, live=None, sel=None,
                     deleted_rows=None, **kw):
    got = g.search(q, k, mode, **kw)
    whole = cdb.DenseIndex(dim=corpus.shape[1], capacity=len(corpus), **(whole_kw or {}))
    whole.append(corpus)
    if deleted_rows is not None:
        assert (whole.delete_rows(deleted_rows.astype(np.uint32)) == 0).all()
    w = whole.batch_search(q, k, mode, **kw)
    whole.close()
    sel = np.arange(len(q)) if sel is None else sel
    want = oracle(corpus, q[sel], k, mode, st, metric, live)
    assert_exact(got, w, want, gid, sel)
    return got


# ----------------------------------------------------------------------------- every final kernel (tests/sharded_plan.py)
def case_corpus(c, seed):
    n, dim = sum(c["shards"]), c["dim"]
    corpus = orc.synth_matrix(seed, n, dim).copy()
    q = orc.synth_matrix(seed + 1, c["nq"], dim).copy()
    if c["crowded"]:
        # 300 copies of one row on every shard: a query equal to it has >= 300 tied candidates, more than prefilter_k
        lay, _ = layout(c["shards"], c["ids"])
        rng = np.random.default_rng(seed)
        block = corpus[lay[0][0]].copy()
        for r0, cnt, _ in lay:
            corpus[r0 + rng.choice(cnt, 300, replace=False)] = block
        q[:c["crowded"]] = block
    return corpus, q


def predicted(c):
    paths = sp.shard_paths(c)
    tensor = [sum(p in ("f16", "s8", "u8") for p, _ in s) for s in paths]
    s8 = [sum(p == "s8" for p, _ in s) for s in paths]
    fb = [1 if c["crowded"] and s[0][0] != "scan" else 0 for s in paths]
    return tensor, s8, fb


@pytest.mark.parametrize("c", [c for c in sp.CASES if c["mode"] != sp.HNSW], ids=lambda c: c["name"])
def test_keys_from_every_final_kernel(c, monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", str(c["ts_s8"]))
    seed = 21000 + sp.CASES.index(c) * 10
    corpus, q = case_corpus(c, seed)
    lay, gid = layout(c["shards"], c["ids"])
    kw = dict(storage_type=ST(c["st"]), metric=MK(c["metric"]))
    g, parts = make_group(corpus, lay, **kw)
    live, deleted_rows = None, None
    if c["deleted"]:
        r0, cnt, _ = lay[-1]
        local = np.sort(np.random.default_rng(seed).choice(cnt, c["deleted"], replace=False)).astype(np.uint32)
        assert (parts[-1].delete_rows(local) == 0).all()
        deleted_rows = local.astype(np.int64) + r0
        live = np.setdiff1d(np.arange(len(corpus)), deleted_rows)
    mode = MODE.BRUTE_RAW if c["mode"] == sp.RAW else MODE.BRUTE_CODES
    before = [p.stats() for p in parts]
    nq = c["nq"]
    sel = np.unique(np.r_[0:min(nq, 8), max(0, sp.CH - 2):min(nq, sp.CH + 2), max(0, nq - 3):nq])
    search_and_check(g, corpus, gid, q, c["k"], mode, ST(c["st"]), MK(c["metric"]), whole_kw=kw, live=live, sel=sel,
                     deleted_rows=deleted_rows, exact_only=c["exact_only"], prefilter_k=c["prefilter_k"],
                     tensor_with_deleted=bool(c["flags"] & sp.TENSOR_WITH_DELETED))
    after = [p.stats() for p in parts]
    tensor, s8, fb = predicted(c)
    assert [a["tensor_searches"] - b["tensor_searches"] for a, b in zip(after, before)] == tensor
    assert [a["s8_searches"] - b["s8_searches"] for a, b in zip(after, before)] == s8
    assert [a["fallbacks"] - b["fallbacks"] for a, b in zip(after, before)] == fb
    if c["crowded"]:
        assert [a["fallback_queries"] for a in after] == [c["crowded"] if f else 0 for f in fb]
    close(g, parts)


@pytest.mark.parametrize("c", [c for c in sp.CASES if c["mode"] == sp.HNSW], ids=lambda c: c["name"])
def test_hnsw_f32_shards_are_the_merge_of_their_own_searches(c):
    dim = c["dim"]
    rng = np.random.default_rng(31)
    n = sum(c["shards"])
    centres = rng.normal(size=(16, dim)).astype(np.float32)
    vecs = (centres[rng.integers(0, 16, n)] + 0.3 * rng.normal(size=(n, dim))).astype(np.float32)
    vecs = (vecs / (np.abs(vecs).max() * 1.01)).astype(np.float32)
    q = (vecs[rng.integers(0, n, c["nq"])] + 0.05 * rng.normal(size=(c["nq"], dim))).astype(np.float32)
    lay, _ = layout(c["shards"], c["ids"])
    g = ShardGroup.local([0] * len(lay))
    parts, per = [], []
    for s, (r0, cnt, base) in enumerate(lay):
        ix = cdb.DenseIndex(dim=dim, storage_type=ST.FullPrecisionFP, capacity=cnt + 1, id_base=base)
        ix.append(vecs[r0:r0 + cnt])
        ix.build_graph(4, 8, 16, 64, 64, 1, 41 + s)
        g.attach(s, ix)
        parts.append(ix)
    kw = dict(ef_search=64, shortlist_size=64)
    for ix in parts:
        per.append(ix.batch_search(q, c["k"], MODE.HNSW, **kw))
    ids, scores, counts, err = g.search(q, c["k"], MODE.HNSW, **kw)
    w_ids, w_scores, w_counts = merge_packed(np.stack([pack_keys(p[0], p[1]) for p in per]), c["k"])
    assert np.array_equal(ids, w_ids) and np.array_equal(bits(scores), bits(w_scores)) and np.array_equal(counts, w_counts)
    assert np.array_equal(err, np.bitwise_or.reduce([p[3] for p in per]))
    assert np.array_equal(counts, np.minimum(c["k"], sum(p[2] for p in per)))          # disjoint shards: nothing lost
    close(g, parts)


# ----------------------------------------------------------------------------- every codes arm
@pytest.mark.parametrize("metric", list(MK), ids=lambda m: m.name)
@pytest.mark.parametrize("st", list(ST), ids=lambda s: s.name)
def test_every_codes_arm_through_the_group(st, metric):
    dim, shards = 40, [900, 1100, 0, 500]
    corpus = orc.synth_matrix(22000 + 7 * int(st) + int(metric), sum(shards), dim)
    q = orc.synth_matrix(22100, 5, dim)
    lay, gid = layout(shards, "desc")
    kw = dict(storage_type=st, metric=metric)
    g, parts = make_group(corpus, lay, **kw)
    want = oracle(corpus, q, 10, MODE.BRUTE_CODES, st, metric)
    if isinstance(want, int):                 # an arm the reference refuses: the group refuses it with the same status
        whole = cdb.DenseIndex(dim=dim, capacity=len(corpus), **kw)
        whole.append(corpus)
        for search in (lambda: whole.batch_search(q, 10, MODE.BRUTE_CODES), lambda: g.search(q, 10, MODE.BRUTE_CODES)):
            with pytest.raises(cdb.CosdataError) as e:
                search()
            assert int(e.value.status) == want
        whole.close()
    else:
        search_and_check(g, corpus, gid, q, 10, MODE.BRUTE_CODES, st, metric, whole_kw=kw)
    close(g, parts)


# ----------------------------------------------------------------------------- ties and signs across shard boundaries
@pytest.mark.parametrize("st,metric", [(None, MK.Cosine), (ST.UnsignedByte, MK.Euclidean), (ST.SubByte3, MK.Hamming),
                                       (ST.UnsignedByte, MK.Hamming), (ST.HalfPrecisionFP, MK.DotProduct),
                                       (ST.BFloat16, MK.Euclidean)])
def test_duplicates_in_other_shards_go_to_the_smaller_id(st, metric):
    # nine distinct rows repeated over four shards; the slot order is the reverse of the id order, so the shard that
    # hands in a tied key first holds the larger ids.  DotProduct: positive rows, negative queries, every score < 0.
    dim, shards = 32, [700, 500, 900, 300]
    base = orc.synth_matrix(22200, 9, dim)
    q = orc.synth_matrix(22201, 6, dim)
    if metric == MK.DotProduct:
        base, q = np.abs(base), -np.abs(q)
    corpus = base[np.random.default_rng(5).integers(0, 9, sum(shards))]
    lay, gid = layout(shards, "desc")
    mode = MODE.BRUTE_RAW if st is None else MODE.BRUTE_CODES
    kw = {} if st is None else dict(storage_type=st, metric=metric)
    g, parts = make_group(corpus, lay, **kw)
    for k in (1, 10, 100, 700):
        ids, scores, counts, err = search_and_check(g, corpus, gid, q, k, mode, st, metric, whole_kw=kw)
        assert (bits(scores[:, 0]) == bits(scores[:, min(k, 100) - 1])).all()       # the top of each query is one tie
        if metric == MK.DotProduct:
            assert (scores < 0).all()
    close(g, parts)


def test_zero_scores_tie_across_shards():
    # raw cosine, query [1, -0, ..., -0], rows with -0 (low-id shard) or +0 (high-id shard) in coordinate 0 and positive
    # values elsewhere: every score is an exact zero, and the group orders them as one index does -- by total_cmp of the
    # score bits the oracle computes, then the smaller id -- whichever slot hands them in first
    dim, shards = 16, [40, 30, 50]
    corpus = np.abs(orc.synth_matrix(22300, sum(shards), dim)) + np.float32(0.125)
    lay, gid = layout(shards, "desc")
    low = lay[-1]                                           # slot 2 holds the smallest ids
    corpus[:, 0] = 0.0
    corpus[low[0]:low[0] + low[1], 0] = -0.0
    q = np.full((3, dim), -0.0, np.float32)
    q[:, 0] = 1.0
    g, parts = make_group(corpus, lay)
    for k in (1, 50, 120):
        ids, scores, _, _ = search_and_check(g, corpus, gid, q, k)
        assert (np.abs(scores) == 0).all()
        key = np.where(bits(scores) >> 31, 0, 1)            # +0 before -0 (total_cmp), each run in ascending id order
        assert (np.diff(key, axis=1) <= 0).all()
        for r in range(len(q)):
            for s in (0, 1):
                run = ids[r][key[r] == s]
                assert (np.diff(run.astype(np.int64)) > 0).all()
    close(g, parts)


# ----------------------------------------------------------------------------- group shapes
@pytest.mark.parametrize("world,k", [(2, 65), (3, 64), (8, 1), (8, 1024), (64, 10)])
def test_wide_groups_with_gaps_empty_shards_and_the_top_of_the_id_range(world, k):
    dim = 24
    rng = np.random.default_rng(world * 1000 + k)
    shards = [int(x) for x in rng.integers(5, 400, world)]
    shards[world // 2 if world > 2 else 0] = 0              # a shard with no rows (not the one holding the top id)
    corpus = orc.synth_matrix(22400 + world, sum(shards), dim)
    q = orc.synth_matrix(22401, 9, dim)
    lay, gid = layout(shards, "desc" if world % 2 else "asc", top=True)
    assert gid.max() == 0xFFFFFFFE
    for st, metric in ((None, MK.Cosine), (ST.UnsignedByte, MK.Euclidean)):
        kw = {} if st is None else dict(storage_type=st, metric=metric)
        g, parts = make_group(corpus, lay, **kw)
        search_and_check(g, corpus, gid, q, k, MODE.BRUTE_RAW if st is None else MODE.BRUTE_CODES, st, metric, whole_kw=kw)
        close(g, parts)


def test_world_64_merge_limit_is_checked_before_any_search():
    dim, world = 16, 64
    assert world * 400 * 8 == sp.MERGE_SMEM_MAX
    shards = [7] * world
    corpus = orc.synth_matrix(22500, sum(shards), dim)
    q = orc.synth_matrix(22501, 3, dim)
    lay, gid = layout(shards, "desc")
    g, parts = make_group(corpus, lay)
    search_and_check(g, corpus, gid, q, 400)              # 64 * 400 keys: exactly 200 KB of shared memory
    stats = [p.stats() for p in parts]
    hist = [p.scan_ms_history().size for p in parts]
    with pytest.raises(cdb.CosdataError) as e:
        g.search(q, 401)
    assert int(e.value.status) == int(cdb.Status.INVALID_PARAMS)
    assert [p.stats() for p in parts] == stats
    assert [p.scan_ms_history().size for p in parts] == hist, "a shard searched before the merge size was refused"
    close(g, parts)


# ----------------------------------------------------------------------------- error bytes, buffer reuse
def test_error_bytes_of_the_last_slot_and_a_clean_search_after():
    dim, shards = 64, [16384, 3000, 2500]
    corpus = orc.synth_matrix(22600, sum(shards), dim).copy()
    lay, gid = layout(shards, "asc")
    corpus[lay[-1][0] + 17] = -1.0                          # all-zero u8 codes, |row| = 0, on the last slot only
    q = orc.synth_matrix(22601, 40, dim)
    kw = dict(storage_type=ST.UnsignedByte, metric=MK.Cosine, keep_raw_f32=True)
    g, parts = make_group(corpus, lay, **kw)
    ids, scores, counts, err = search_and_check(g, corpus, gid, q, 12, MODE.BRUTE_CODES, ST.UnsignedByte, MK.Cosine, whole_kw=kw)
    assert err.all(), "the flag of the last slot did not reach the merge"
    # smaller batch and k, raw rows (no zero magnitude): nothing of the first search may survive in the gather buffer
    ids, scores, counts, err = search_and_check(g, corpus, gid, q[:7], 5, whole_kw=kw)
    assert not err.any()
    close(g, parts)


# ----------------------------------------------------------------------------- the device form
def test_rank_group_of_one_on_a_side_stream_equals_the_host_form():
    import torch
    dim, n, nq, k = 64, 20000, 2051, 16
    corpus = orc.synth_matrix(22700, n, dim)
    q = orc.synth_matrix(22701, nq, dim)
    g = ShardGroup.rank(None, 1, 0, 0)
    ix = cdb.DenseIndex(dim=dim, capacity=n, id_base=77)
    ix.append(corpus)
    g.attach(0, ix)
    h_ids, h_scores, h_counts, h_err = g.search(q, k)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dq = torch.from_numpy(q).cuda()
        d_ids = torch.full((nq, k), -1, dtype=torch.int32, device="cuda")
        d_scores = torch.full((nq, k), 7.0, dtype=torch.float32, device="cuda")
        d_counts = torch.zeros(nq, dtype=torch.int32, device="cuda")
        d_err = torch.full((nq,), 9, dtype=torch.uint8, device="cuda")
    g.search_device(dq.data_ptr(), nq, k, d_ids.data_ptr(), d_scores.data_ptr(), d_counts.data_ptr(), d_err.data_ptr(),
                    stream_ptr=s.cuda_stream)
    s.synchronize()
    assert np.array_equal(d_ids.cpu().numpy().view(np.uint32), h_ids)
    assert np.array_equal(bits(d_scores.cpu().numpy()), bits(h_scores))
    assert np.array_equal(d_counts.cpu().numpy().view(np.uint32), h_counts) and np.array_equal(d_err.cpu().numpy(), h_err)
    want_ids, want_scores = orc.brute_topk_f32(corpus, q[-4:], k)
    assert np.array_equal(h_ids[-4:], want_ids + np.uint32(77)) and np.array_equal(bits(h_scores[-4:]), bits(want_scores))
    close(g, [ix])


# ----------------------------------------------------------------------------- attach checks
@pytest.mark.parametrize("field", ["dim", "metric", "storage_type", "id_range"])
def test_attach_refuses_a_shard_unlike_an_attached_one_in_either_order(field):
    a_kw = dict(dim=64, storage_type=ST.UnsignedByte, metric=MK.Cosine, capacity=100, id_base=100)
    b_kw = dict(a_kw, id_base=200)
    b_kw.update({"dim": dict(dim=128), "metric": dict(metric=MK.Euclidean), "storage_type": dict(storage_type=ST.SubByte2),
                 "id_range": dict(id_base=150)}[field])
    for order in ((1, 0), (0, 1)):                         # the second attach must fail, whichever slot came first
        g = ShardGroup.local([0, 0])
        a, b = cdb.DenseIndex(**a_kw), cdb.DenseIndex(**b_kw)
        g.attach(order[0], a)
        with pytest.raises(cdb.CosdataError) as e:
            g.attach(order[1], b)
        assert int(e.value.status) == int(cdb.Status.INVALID_PARAMS)
        assert field.split("_")[0] in str(e.value)
        close(g, [a, b])
