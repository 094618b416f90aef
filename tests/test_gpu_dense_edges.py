"""The dense exact paths at their plan and arithmetic edges: the exact scan (scan.cu) over every template and merge branch
it plans, the pairwise scorers (scorers.cuh) at their loop boundaries, the quantizer's two magnitude kernels
(quantize.cu) and the chunked f32 re-rank (pairs.cu).  Every comparison with the CPU oracle is bit-exact: ids, counts and
error bytes with array_equal, f32 scores on their raw bits."""
import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc

pytestmark = pytest.mark.gpu
ST, MK = cdb.StorageType, cdb.DistanceMetricKind
SUB = (ST.SubByte1, ST.SubByte2, ST.SubByte3)
CHUNK = 2048                      # queries per search chunk (search_device_locked)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def rup(x, m):
    return (x + m - 1) // m * m


def row_pitch(st, dim):
    """bytes per stored row (common.cuh row_pitch_bytes); st None = raw f32 rows"""
    if st is None or st == ST.FullPrecisionFP:
        return rup(4 * dim, 16)
    if st == ST.UnsignedByte:
        return dim if dim % 16 == 0 else rup(dim, 16)
    if st in SUB:
        return int(st) * rup((dim + 7) // 8, 16)
    return rup(2 * dim, 16)


# ------------------------------------------------------------------ the exact scan's plan, restated from scan.cu
SCAN_THREADS = 256                # threads per CTA
RPP = 256                         # rows per pass per CTA
QB_BUDGET = 100 * 1024            # pick_qb: shared-memory budget of one query group
MAX_KEYS = 8192                   # scan_plan_nsplit: at most 8192 / k splits
MAX_SPLIT = 1024
MERGE_RANK_MAX = 768              # merge_partials_kernel: rank selection up to nsplit * k = 768 keys, bitonic sort above


def topk_smem_bytes(qb, k):
    return qb * (8 + 4 + 4) + qb * (k + 3 * RPP + k) * 8 + 16


def pick_qb(nq, pitch, k):
    qb = 8 if nq >= 5 else (4 if nq >= 3 else (2 if nq == 2 else 1))
    while qb > 1 and qb * pitch + topk_smem_bytes(qb, k) + 64 > QB_BUDGET:
        qb >>= 1
    return qb


def scan_smem(qb, pitch, k):
    return qb * pitch + ((qb + 3) & ~3) * 4 + topk_smem_bytes(qb, k)


def scan_plan_nsplit(nq, n, pitch, k, sms):
    qb = pick_qb(nq, pitch, k)
    ngroups = (nq + qb - 1) // qb
    npass = (n + RPP - 1) // RPP
    resident = 2 * sms
    max_split = max(npass, 1)
    if max_split > MAX_KEYS // k:
        max_split = MAX_KEYS // k or 1
    max_split = min(max_split, MAX_SPLIT)
    best, best_score = 1, -1.0
    for s in range(1, max_split + 1):
        total = s * ngroups
        waves = (total + resident - 1) // resident
        eff = total / (waves * resident)
        if waves > 8:
            eff *= 8.0 / waves
        if npass // s < 4 and s > 1:
            eff *= 0.5
        if eff > best_score + 1e-9:
            best_score, best = eff, s
    return best


def scan_plan(st, metric, dim, n, nq, k, sms):
    """-> (kernel, QB, merge branch) of every 2048-query chunk of one exact search; st None = BRUTE_RAW"""
    pitch = row_pitch(st, dim)
    f32 = st is None or (st == ST.FullPrecisionFP and metric == MK.Cosine)
    out = []
    for off in range(0, nq, CHUNK):
        m = min(CHUNK, nq - off)
        qb = pick_qb(m, pitch, k)
        nsplit = scan_plan_nsplit(m, n, pitch, k, sms)
        out.append(("f32" if f32 else "generic", qb, "rank" if nsplit * k <= MERGE_RANK_MAX else "bitonic"))
    return out


def arm_ok(metric, st):
    if metric in (MK.Cosine,):
        return True
    if metric == MK.DotProduct:
        return st != ST.FullPrecisionFP
    if metric == MK.Euclidean:
        return st in (ST.UnsignedByte, ST.HalfPrecisionFP, ST.BFloat16)
    return st != ST.FullPrecisionFP


# (storage or None for BRUTE_RAW, metric, dim, n, nq, k)
PLAN_CASES = (
    # nq-driven QB on both kernels
    [(None, MK.Cosine, 64, 3000, nq, 10) for nq in (1, 2, 3, 4, 5, 9, 17)]
    + [(ST.UnsignedByte, MK.Euclidean, 100, 2500, nq, 10) for nq in (1, 2, 3, 4, 5, 9, 17)]
    + [(ST.SubByte3, MK.Hamming, 100, 2500, nq, 10) for nq in (1, 2, 3, 5)]
    # k-driven shrink: k 1024 allows at most QB 4, and QB 2 at 3 KB rows
    + [(None, MK.Cosine, 64, 5000, 5, 1024), (None, MK.Cosine, 768, 3000, 5, 1024),
       (ST.UnsignedByte, MK.Hamming, 64, 5000, 5, 1024), (ST.UnsignedByte, MK.Euclidean, 3072, 3000, 5, 1024)]
    # row-driven shrink: 8 rows of f32 codes (or u8) past the 100 KB budget
    + [(ST.FullPrecisionFP, MK.Cosine, d, 1000, 9, 10) for d in (3300, 6000, 12000)]
    + [(ST.UnsignedByte, MK.Euclidean, d, 700, 9, 10) for d in (13000, 30000, 60000)]
    # every (metric, storage) arm, once per merge branch
    + [(st, m, 100, 2500, 5, 10) for m in MK for st in ST]
    + [(st, m, 37, 20000, 3, 100) for m in MK for st in ST]
    + [(None, MK.Cosine, 40, 20000, 3, 100)]
)


def case_id(c):
    st, m, dim, n, nq, k = c
    return f"{'raw' if st is None else st.name}-{m.name}-d{dim}-n{n}-q{nq}-k{k}"


def test_plan_matrix_covers_every_template_and_merge_branch():
    sms = sm_count()
    kernels, merges = set(), set()
    for st, m, dim, n, nq, k in PLAN_CASES:
        if st is not None and not arm_ok(m, st):
            continue
        for kern, qb, branch in scan_plan(st, m, dim, n, nq, k, sms):
            kernels.add((kern, qb))
            merges.add((m, branch))
    assert kernels == {(kern, qb) for kern in ("f32", "generic") for qb in (1, 2, 4, 8)}, sorted(kernels)
    assert merges == {(m, b) for m in MK for b in ("rank", "bitonic")}, sorted(merges)
    # the k- and row-driven shrinks happen where intended
    assert pick_qb(5, row_pitch(None, 64), 1024) == 4 and pick_qb(5, row_pitch(None, 768), 1024) == 2
    assert 8 * row_pitch(ST.FullPrecisionFP, 3300) > QB_BUDGET


def search_codes_vs_oracle(ix, st, metric, dim, corpus_codes, mags, q, k, id_base=0, **kw):
    qc, qm = orc.quantize_batch(int(st), q)
    rc, want_ids, want_scores, want_err = orc.brute_topk_codes(int(metric), int(st), dim, corpus_codes, mags, qc, qm, k)
    if rc != 0:                       # StorageMismatch / unimplemented arm: the whole search is an Err
        with pytest.raises(cdb.CosdataError) as e:
            ix.batch_search(q, k, cdb.SearchMode.BRUTE_CODES, **kw)
        assert int(e.value.status) == rc
        return None
    ids, scores, counts, err = ix.batch_search(q, k, cdb.SearchMode.BRUTE_CODES, **kw)
    want_ids = np.where(want_ids == cdb.INVALID_ID, want_ids, want_ids + np.uint32(id_base))
    assert np.array_equal(ids, want_ids), "top-k ids differ from the oracle"
    assert np.array_equal(bits(scores), bits(want_scores)), "scores not bit-identical"
    assert np.array_equal(err, want_err)
    assert np.array_equal(counts, (want_ids != cdb.INVALID_ID).sum(axis=1).astype(np.uint32))   # rows a query could score
    return ids, scores


def search_raw_vs_oracle(ix, corpus, q, k, id_base=0, **kw):
    ids, scores, counts, err = ix.batch_search(q, k, cdb.SearchMode.BRUTE_RAW, **kw)
    want_ids, want_scores = orc.brute_topk_f32(corpus, q, k)
    want_ids = np.where(want_ids == cdb.INVALID_ID, want_ids, want_ids + np.uint32(id_base))
    assert np.array_equal(ids, want_ids), "top-k ids differ from the oracle"
    assert np.array_equal(bits(scores), bits(want_scores)), "scores not bit-identical"
    assert np.array_equal(counts, np.full(len(q), min(k, corpus.shape[0]), np.uint32))
    return ids, scores


def run_case(st, metric, dim, corpus, q, k, id_base=0, **kw):
    n = corpus.shape[0]
    if st is None:
        ix = cdb.DenseIndex(dim=dim, capacity=n, id_base=id_base)
        ix.append(corpus)
        out = search_raw_vs_oracle(ix, corpus, q, k, id_base, **kw)
    else:
        ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n, id_base=id_base)
        ix.append(corpus)
        codes, mags = orc.quantize_batch(int(st), corpus)
        out = search_codes_vs_oracle(ix, st, metric, dim, codes, mags, q, k, id_base, **kw)
    ix.close()
    return out


@pytest.mark.parametrize("case", PLAN_CASES, ids=case_id)
def test_scan_plan_case_matches_oracle(case):
    st, metric, dim, n, nq, k = case
    seed = 11000 + dim + nq + k + (0 if st is None else 97 * int(st)) + 13 * int(metric)
    corpus = orc.synth_matrix(seed, n, dim)
    q = orc.synth_matrix(seed + 1, nq, dim)
    run_case(st, metric, dim, corpus, q, k)


# ------------------------------------------------------------------ row counts, ties, ids, deleted rows, batches
@pytest.mark.parametrize("n", [255, 256, 257, 511, 512, 513, 10239, 10240, 10241])
@pytest.mark.parametrize("st,metric", [(None, MK.Cosine), (ST.UnsignedByte, MK.Euclidean), (ST.SubByte3, MK.Hamming),
                                       (ST.BFloat16, MK.DotProduct)])
def test_row_count_edges(st, metric, n):
    dim = 24
    corpus = orc.synth_matrix(12000 + n, n, dim)
    q = orc.synth_matrix(12001, 5, dim)
    for k in (1, 10, 300):
        run_case(st, metric, dim, corpus, q, k)


@pytest.mark.parametrize("st,metric", [(None, MK.Cosine), (ST.UnsignedByte, MK.Euclidean), (ST.SubByte2, MK.Hamming)])
def test_fewer_rows_than_k_and_as_many(st, metric):
    dim = 24
    q = orc.synth_matrix(12101, 3, dim)
    for n, k in ((5, 10), (10, 10), (1, 1), (700, 700), (300, 1024)):
        run_case(st, metric, dim, orc.synth_matrix(12100 + n, n, dim), q, k)


@pytest.mark.parametrize("st,metric", [(None, MK.Cosine), (ST.UnsignedByte, MK.DotProduct), (ST.UnsignedByte, MK.Euclidean),
                                       (ST.SubByte1, MK.Hamming), (ST.SubByte2, MK.Cosine), (ST.HalfPrecisionFP, MK.Hamming)])
def test_integer_ties_across_splits_and_passes(st, metric):
    # nine distinct rows repeated at random over 20000 rows: every score ties with thousands of copies in other passes
    # and other splits, and the smaller id must win each tie
    dim, n = 48, 20000
    base = orc.synth_matrix(12200, 9, dim)
    corpus = base[np.random.default_rng(3).integers(0, 9, n)]
    q = orc.synth_matrix(12201, 5, dim)
    for k in (1, 10, 100, 1000):
        ids, scores = run_case(st, metric, dim, corpus, q, k, exact_only=True)
        if k >= 10:
            assert (bits(scores[:, 0]) == bits(scores[:, 9])).all()      # the top 10 of each query is one tie


@pytest.mark.parametrize("st,metric", [(None, MK.Cosine), (ST.UnsignedByte, MK.Euclidean), (ST.SubByte3, MK.Hamming)])
def test_id_base_at_the_top_of_the_id_range(st, metric):
    dim, n = 32, 3000
    id_base = 2**32 - n - 1                    # the last row is id 0xFFFFFFFE
    corpus = orc.synth_matrix(12300, n, dim)
    q = corpus[[n - 1, 0, 1234]].copy()
    for k in (10, 300):
        ids, _ = run_case(st, metric, dim, corpus, q, k, id_base=id_base)
        assert (ids != cdb.INVALID_ID).all() and ids.max() <= 0xFFFFFFFE


@pytest.mark.parametrize("st,metric", [(ST.UnsignedByte, MK.Euclidean), (ST.HalfPrecisionFP, MK.Euclidean),
                                       (ST.UnsignedByte, MK.Hamming), (ST.SubByte2, MK.Hamming)])
def test_deleted_rows_are_skipped_by_the_exact_scan(st, metric):
    dim, n = 64, 5000
    corpus = orc.synth_matrix(12400 + int(st), n, dim)
    q = np.concatenate([corpus[[0, 4999, 600]], orc.synth_matrix(12401, 4, dim)])
    codes, mags = orc.quantize_batch(int(st), corpus)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n)
    ix.append(corpus)
    rng = np.random.default_rng(4)
    dead = np.unique(np.concatenate([[0, 4999], np.arange(512, 768), rng.choice(n, 500, replace=False)]))
    gone = np.zeros(0, np.int64)
    for live in (np.setdiff1d(np.arange(n), dead), np.array([3, 777, 2048, 4000, 4998])):   # then all but five rows
        todo = np.setdiff1d(np.setdiff1d(np.arange(n), live), gone)
        assert (np.asarray(ix.delete_rows(todo.astype(np.uint32))) == 0).all()
        gone = np.union1d(gone, todo)
        qc, qm = orc.quantize_batch(int(st), q)
        for k in (10, 300):
            rc, want_ids, want_scores, want_err = orc.brute_topk_codes(int(metric), int(st), dim, codes[live], mags[live], qc, qm, k)
            assert rc == 0
            want_ids = np.where(want_ids == cdb.INVALID_ID, want_ids, live[np.minimum(want_ids, live.size - 1)].astype(np.uint32))
            ids, scores, counts, err = ix.batch_search(q, k, cdb.SearchMode.BRUTE_CODES)
            assert np.array_equal(ids, want_ids) and np.array_equal(bits(scores), bits(want_scores))
            assert np.array_equal(counts, np.full(len(q), min(k, live.size), np.uint32)) and np.array_equal(err, want_err)
    ix.close()


@pytest.mark.parametrize("st,metric", [(None, MK.Cosine), (ST.UnsignedByte, MK.Euclidean)])
def test_batch_of_three_chunks(st, metric):
    dim, n, nq = 32, 3000, 4100
    corpus = orc.synth_matrix(12500, n, dim)
    q = orc.synth_matrix(12501, nq, dim)
    for k in (1, 64):
        run_case(st, metric, dim, corpus, q, k)


@pytest.mark.parametrize("metric", [MK.Cosine, MK.DotProduct])
@pytest.mark.parametrize("st", [ST.UnsignedByte, ST.SubByte2])
def test_exact_only_answers_shapes_of_the_u8_tensor_path(st, metric):
    dim, n = 96, 16500
    corpus = orc.synth_matrix(12600 + int(st), n, dim)
    codes, mags = orc.quantize_batch(int(st), corpus)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n)
    ix.append(corpus)
    for nq in (1, 5, 130):
        q = orc.synth_matrix(12601 + nq, nq, dim)
        before = ix.stats()["tensor_searches"]
        search_codes_vs_oracle(ix, st, metric, dim, codes, mags, q, 10, exact_only=True)
        assert ix.stats()["tensor_searches"] == before
    ix.close()


# ------------------------------------------------------------------ scorer loop boundaries
# dot16_seq: 64-element blocks, 8-element steps, scalar tail; dot_u8_int: 64-byte blocks, 4-byte steps, byte tail;
# sub-byte scorers: plane_bytes = ceil(D / 8) with every remainder mod 4
SCORER_DIMS = [1, 7, 8, 9, 23, 31, 50, 63, 64, 65, 71, 127, 129, 1023, 1025]


def test_scorer_dims_reach_every_sub_byte_word_remainder():
    assert {((d + 7) // 8) % 4 for d in SCORER_DIMS} == {0, 1, 2, 3}


def scorer_rows(seed, n, dim):
    m = orc.synth_matrix(seed, n, dim).copy()
    m[0] = 1.0                                              # saturated codes
    m[1] = -1.0
    m[2, ::2] = 1.0
    if n > 3:
        m[3] = 0.0                                          # zero norm
    return m


@pytest.mark.parametrize("dim", SCORER_DIMS)
@pytest.mark.parametrize("st", list(ST))
def test_scorer_boundaries(st, dim):
    n = 40
    x = scorer_rows(13000 + dim, n, dim)
    y = scorer_rows(13100 + dim, n, dim)[::-1].copy()
    xc, xm = orc.quantize_batch(int(st), x)
    yc, ym = orc.quantize_batch(int(st), y)
    for metric in MK:
        got, status = cdb.DistanceMetric(metric).calculate_pairs(st, dim, xc, xm, yc, ym)
        for i in range(n):
            rc, v = orc.distance(int(metric), int(st), dim, xc[i], xm[i], yc[i], ym[i])
            assert status[i] == rc, (metric, i, status[i], rc)
            if rc == 0:
                assert bits(got[i]) == bits(v), (metric, i, got[i], v)
        ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n)
        ix.append(y)
        ids = np.array([0, 1, 2, 3, n - 1, 17, 17], dtype=np.uint32)
        for qi in (0, 2, 5):
            got, status = ix.score_ids(x[qi], ids)
            for j, r in enumerate(ids):
                rc, v = orc.distance(int(metric), int(st), dim, xc[qi], xm[qi], yc[r], ym[r])
                assert status[j] == rc and (rc != 0 or bits(got[j]) == bits(v)), (metric, qi, r)
        search_codes_vs_oracle(ix, st, metric, dim, yc, ym, x[:6], 10)
        ix.close()


def f16_like_codes(st, rng, n, dim):
    """u16 codes mixing subnormals, the largest finite magnitude and ordinary values; largest-magnitude entries are
    placed where the other operand holds the same value, so no product is -inf against a +inf"""
    top = 0x7BFF if st == ST.HalfPrecisionFP else 0x7F7F
    one = 0x3C00 if st == ST.HalfPrecisionFP else 0x3F80
    normal = rng.integers(one - 0x0800, one + 0x0400, (n, dim)).astype(np.uint16)
    sub = rng.integers(1, 0x03FF if st == ST.HalfPrecisionFP else 0x007F, (n, dim)).astype(np.uint16)
    kind = rng.integers(0, 3, (n, dim))
    c = np.where(kind == 0, sub, normal).astype(np.uint16)
    c |= (rng.integers(0, 2, (n, dim)) << 15).astype(np.uint16)
    big = np.zeros((n, dim), bool)
    big[::2, ::5] = True                                  # even rows only: an overflowing bf16 product swamps the sum
    return c, big, top


@pytest.mark.parametrize("dim", [9, 64, 71, 129])
@pytest.mark.parametrize("st", [ST.HalfPrecisionFP, ST.BFloat16])
def test_f16_bf16_subnormal_and_largest_operands(st, dim):
    rng = np.random.default_rng(dim + int(st))
    n = 32
    xc, big, top = f16_like_codes(st, rng, n, dim)
    yc, _, _ = f16_like_codes(st, rng, n, dim)
    sign = (rng.integers(0, 2, (n, dim)) << 15).astype(np.uint16)
    xc[big] = top | sign[big]
    yc[big] = top | sign[big]
    yc[: n // 2, 1::5] = xc[: n // 2, 1::5] & 0x807F          # subnormal against normal/large on half of the rows
    xm = np.abs(orc.synth_matrix(14000 + dim, 1, n)[0]) + np.float32(0.5)
    ym = np.abs(orc.synth_matrix(14001 + dim, 1, n)[0]) + np.float32(0.5)
    xb, yb = xc.view(np.uint8).reshape(n, 2 * dim), yc.view(np.uint8).reshape(n, 2 * dim)
    for metric in MK:
        got, status = cdb.DistanceMetric(metric).calculate_pairs(st, dim, xb, xm, yb, ym)
        for i in range(n):
            rc, v = orc.distance(int(metric), int(st), dim, xb[i], xm[i], yb[i], ym[i])
            assert status[i] == rc
            if rc == 0:
                assert bits(got[i]) == bits(v), (metric, i, got[i], v)


U8_WRAP_DIM = 140_000


def u8_wrap_rows(dim):
    """saturated rows (every code 255) and mixed rows; at D = 140,000 both half-sums of dot_product_u8 pass 2^32"""
    rng = np.random.default_rng(7)
    rows = [np.ones(dim, np.float32) for _ in range(3)]
    for frac in (0.999, 0.99, 0.9, 0.75, 0.5, 0.3):
        r = np.ones(dim, np.float32)
        r[rng.random(dim) > frac] = -1.0                       # code 0
        rows.append(r)
    r = np.ones(dim, np.float32)
    r[: dim // 2] = 0.5
    rows.append(r)
    rows.append(orc.synth_matrix(15000, 1, dim)[0])
    return np.stack(rows)


def test_u8_dot_wraps_like_the_reference():
    dim = U8_WRAP_DIM
    corpus = u8_wrap_rows(dim)
    n = corpus.shape[0]
    q = corpus[[0, 5, 9]].copy()
    codes, mags = orc.quantize_batch(int(ST.UnsignedByte), corpus)
    qc, qm = orc.quantize_batch(int(ST.UnsignedByte), q)
    exact = int(codes[0].astype(np.int64) @ codes[0].astype(np.int64))
    assert exact > 2**33 and orc.distance(int(MK.DotProduct), 0, dim, codes[0], mags[0], codes[0], mags[0])[1] != np.float32(exact)
    assert mags[0] != np.float32(np.sqrt(exact))                 # the u32 sum of squares wraps too
    got, status = cdb.DistanceMetric(MK.DotProduct).calculate_pairs(ST.UnsignedByte, dim, codes, mags, codes[::-1].copy(),
                                                                    mags[::-1].copy())
    for i in range(n):
        rc, v = orc.distance(int(MK.DotProduct), 0, dim, codes[i], mags[i], codes[n - 1 - i], mags[n - 1 - i])
        assert status[i] == rc == 0 and bits(got[i]) == bits(v), (i, got[i], v)
    for metric in (MK.Cosine, MK.DotProduct):
        ix = cdb.DenseIndex(dim=dim, storage_type=ST.UnsignedByte, metric=metric, capacity=n)
        ix.append(corpus)
        got_codes, got_mags = ix.read_codes(0, n)
        assert np.array_equal(got_codes, codes) and np.array_equal(bits(got_mags), bits(mags))
        rc, want_ids, want_scores, want_err = orc.brute_topk_codes(int(metric), 0, dim, codes, mags, qc, qm, n)
        ids, scores, counts, err = ix.batch_search(q, n, cdb.SearchMode.BRUTE_CODES)
        assert np.array_equal(ids, want_ids), "ranking differs from the oracle's wrapped dot products"
        assert np.array_equal(bits(scores), bits(want_scores)), "scores differ from the oracle's wrapped dot products"
        got, status = ix.score_ids(q[0], np.arange(n, dtype=np.uint32))
        for r in range(n):
            rc, v = orc.distance(int(metric), 0, dim, qc[0], qm[0], codes[r], mags[r])
            assert status[r] == rc and bits(got[r]) == bits(v), (metric, r)
        ix.close()


# ------------------------------------------------------------------ quantizer
def mags_route(n, dim):
    """quantize.cu run_quantize: one CTA per row for small batches whose squares fit 48 KB, one thread per row otherwise"""
    return "cta" if n <= 8192 and dim * 4 + 16 <= 48 * 1024 else "thread"


QUANT_SHAPES = [(8192, 96), (8193, 96), (9, 12284), (9, 12285)]


def test_quant_shapes_reach_both_magnitude_kernels():
    assert {mags_route(n, d) for n, d in QUANT_SHAPES} == {"cta", "thread"}
    assert mags_route(8192, 12284) == "cta" and mags_route(8193, 12284) == "thread" and mags_route(8192, 12285) == "thread"


def nxt(x, toward):
    return np.nextafter(np.float32(x), np.float32(toward))


def edge_values(lo, hi):
    v = [np.nan, np.inf, -np.inf, 0.0, -0.0, lo, hi, nxt(lo, -np.inf), nxt(lo, np.inf), nxt(hi, -np.inf), nxt(hi, np.inf)]
    for r in (1, 2, 3):                                   # sub-byte step boundaries -1 + j * 2 / 2^r and their neighbours
        for j in range(2**r + 1):
            b = np.float32(-1.0 + j * 2.0 / 2**r)
            v += [b, nxt(b, -np.inf), nxt(b, np.inf)]
    e = 2.0 ** -11                                        # f16 ties (to even) in the normal and subnormal range, overflow
    v += [1 + e, 1 + 3 * e, -(1 + e), 2.0**-25, 3 * 2.0**-25, 65520.0, nxt(65520.0, 0), 65504.0, 2.0**-14 + 2.0**-25]
    e = 2.0 ** -8                                         # bf16 ties
    v += [1 + e, 1 + 3 * e, -(1 + 3 * e), 3.3895314e38, np.finfo(np.float32).max, 1e-40, -1e-45]
    return np.array(v, np.float32)


def quant_matrix(n, dim, lo, hi, seed):
    m = orc.synth_matrix(seed, n, dim).copy()
    ev = edge_values(lo, hi)
    for r in range(min(n, 5)):                            # the edge values at every offset class of a 4-byte word
        row = np.resize(np.roll(ev, r), dim)
        m[(r * 1237) % n] = row
    return m


def same_mags(got, want):
    """bits equal; a row holding a NaN has a NaN magnitude whose payload the reference does not fix"""
    both_nan = np.isnan(got) & np.isnan(want)
    return np.array_equal(bits(got)[~both_nan], bits(want)[~both_nan]) and np.array_equal(np.isnan(got), np.isnan(want))


@pytest.mark.parametrize("n,dim", QUANT_SHAPES)
@pytest.mark.parametrize("st", list(ST))
def test_quantize_append_and_append_device_match_oracle(st, n, dim):
    import torch
    lo, hi = (-0.8, 0.9) if st == ST.UnsignedByte else (-1.0, 1.0)
    m = quant_matrix(n, dim, lo, hi, 16000 + n + dim)
    want_c, want_m = orc.quantize_batch(int(st), m, lo, hi)
    codes, mags = cdb.ScalarQuantization().quantize_batch(m, st, (lo, hi))
    assert np.array_equal(codes, want_c), "quantize_batch codes"
    assert same_mags(mags, want_m), "quantize_batch magnitudes"
    for dev in (False, True):
        ix = cdb.DenseIndex(dim=dim, storage_type=st, capacity=n, value_range=(lo, hi))
        if dev:
            d = torch.from_numpy(m).cuda()
            ix.append_device(d.data_ptr(), n)
            torch.cuda.synchronize()
        else:
            ix.append(m)
        codes, mags = ix.read_codes(0, n)
        assert np.array_equal(codes, want_c), ("codes", dev)
        assert same_mags(mags, want_m), ("magnitudes", dev)
        ix.close()


@pytest.mark.parametrize("st", list(ST))
def test_quantize_with_an_empty_range(st):
    m = quant_matrix(6, 40, 0.5, 0.5, 16100)
    want_c, want_m = orc.quantize_batch(int(st), m, 0.5, 0.5)
    codes, mags = cdb.ScalarQuantization().quantize_batch(m, st, (0.5, 0.5))
    assert np.array_equal(codes, want_c) and same_mags(mags, want_m)


def test_u8_magnitudes_wrap_at_140000():
    dim = U8_WRAP_DIM
    corpus = u8_wrap_rows(dim)
    want_c, want_m = orc.quantize_batch(int(ST.UnsignedByte), corpus)
    assert mags_route(corpus.shape[0], dim) == "thread"
    codes, mags = cdb.ScalarQuantization().quantize_batch(corpus, ST.UnsignedByte)
    assert np.array_equal(codes, want_c) and np.array_equal(bits(mags), bits(want_m))


# ------------------------------------------------------------------ re-rank (cdb_rerank_f32)
RERANK_BUF = 2048                 # pairs.cu: keys per chunk


@pytest.fixture(scope="module")
def rerank_index():
    dim, n = 64, 20000
    corpus = orc.synth_matrix(17000, n, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(corpus)
    yield ix, corpus
    ix.close()


def rerank_vs_oracle(ix, corpus, q, cand, k, id_base=0):
    ids, scores, cnt = ix.rerank(q, cand + np.uint32(id_base), k)
    want_ids, want_scores = orc.rerank_f32(corpus, q, cand, k)
    want_ids = np.where(want_ids == cdb.INVALID_ID, want_ids, want_ids + np.uint32(id_base))
    assert cnt == min(k, cand.size)
    assert np.array_equal(ids, want_ids), "re-ranked ids differ from the oracle"
    assert np.array_equal(bits(scores), bits(want_scores)), "re-ranked scores not bit-identical"
    return ids


@pytest.mark.parametrize("k", [1, 10, 64, 960, 1024])
@pytest.mark.parametrize("ncand", [2047, 2048, 2049, 5000, 20000])
def test_rerank_chunks(rerank_index, ncand, k):
    ix, corpus = rerank_index
    q = orc.synth_matrix(17001 + k, 1, corpus.shape[1])[0]
    cand = np.random.default_rng(ncand + k).permutation(corpus.shape[0])[:ncand].astype(np.uint32)
    rerank_vs_oracle(ix, corpus, q, cand, k)


@pytest.mark.parametrize("group", [2, 64, 65])
@pytest.mark.parametrize("spread", ["one_chunk", "across_chunks"])
def test_rerank_keeps_every_listed_copy(rerank_index, group, spread):
    ix, corpus = rerank_index
    q = orc.synth_matrix(17100, 1, corpus.shape[1])[0]
    rng = np.random.default_rng(group)
    base = rng.permutation(corpus.shape[0])[:5000].astype(np.uint32)
    best = orc.rerank_f32(corpus, q, base, 3)[0]
    cand = base[~np.isin(base, best)]
    for w, winner in enumerate(best):                       # `group` copies of each of the three best candidates
        if spread == "one_chunk":
            pos = 100 + w * 300 + np.arange(group)
        else:
            pos = np.linspace(w, cand.size - 1, group).astype(np.int64)
        cand = np.insert(cand, np.sort(pos), winner)
    assert np.count_nonzero(cand == best[0]) == group
    if spread == "one_chunk":
        assert (np.nonzero(cand == best[0])[0] < RERANK_BUF).all()
    else:
        assert len({p // RERANK_BUF for p in np.nonzero(cand == best[0])[0]}) > 1
    for k in (1, 10, 64, 200, 1024):
        ids = rerank_vs_oracle(ix, corpus, q, cand, k)
        assert np.count_nonzero(ids == best[0]) == min(k, group)


def test_rerank_refuses_ids_outside_the_index():
    dim, n, id_base = 32, 500, 1000
    corpus = orc.synth_matrix(17200, n, dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n + 10, id_base=id_base)
    ix.append(corpus)
    q = orc.synth_matrix(17201, 1, dim)[0]
    cand = np.arange(0, n, 7, dtype=np.uint32)
    rerank_vs_oracle(ix, corpus, q, cand, 10, id_base)
    for bad in (id_base + n, id_base + n + 5, id_base - 1, 0, cdb.INVALID_ID):
        with pytest.raises(cdb.CosdataError) as e:
            ix.rerank(q, np.append(cand + id_base, np.uint32(bad)).astype(np.uint32), 10)
        assert e.value.status == cdb.Status.INVALID_PARAMS
    rerank_vs_oracle(ix, corpus, q, cand, 10, id_base)      # the index still answers
    ix.close()


# ------------------------------------------------------------------ the exact scan's shared-memory limit
def optin_smem():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def largest_raw_dim(k):
    """largest multiple of 4 whose one-query plan (pick_qb shrinks a wide row to QB 1) fits the per-block limit"""
    lim = optin_smem()
    d = (lim - scan_smem(1, 0, k)) // 4 // 4 * 4
    assert scan_smem(1, row_pitch(None, d), k) <= lim < scan_smem(1, row_pitch(None, d + 4), k)
    return d


@pytest.mark.parametrize("k,smaller_k", [(10, 1), (1024, 10)])
def test_exact_scan_refuses_rows_past_the_shared_memory_limit(k, smaller_k):
    d = largest_raw_dim(k)
    n = k + 37
    q = orc.synth_matrix(18001, 2, d + 4)
    corpus = orc.synth_matrix(18000, n, d + 4)
    # the largest dimension that fits is answered
    fit = np.ascontiguousarray(corpus[:, :d])
    ix = cdb.DenseIndex(dim=d, capacity=n)
    ix.append(fit)
    search_raw_vs_oracle(ix, fit, np.ascontiguousarray(q[:, :d]), k)
    ix.close()
    # four more floats are refused with a message, and the same index still answers a plan that fits
    ix = cdb.DenseIndex(dim=d + 4, capacity=n)
    ix.append(corpus)
    with pytest.raises(cdb.CosdataError) as e:
        ix.batch_search(q, k)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    assert str(d + 4) in str(e.value) and f"k {k}" in str(e.value)
    assert scan_smem(1, row_pitch(None, d + 4), smaller_k) <= optin_smem()
    search_raw_vs_oracle(ix, corpus, q, smaller_k)
    ix.close()
