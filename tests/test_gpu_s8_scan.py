"""The s8 prefilter scan (csrc/tensor_scan.cu, KIND 2; DESIGN.md section 5c) against an exact model of its filter.

The s8 filter can be modelled exactly: dp is an s32 dot product of codes that numpy reproduces bit for bit
(tests/prefilter_s8.py), and the kernels document when they read the bound -- every CTA of the main pass starts from the
seeding pass's class maxima, and the bound only rises from there, up to the k-th class maximum over all rows.  So per
query the number of candidates the scan emits is bracketed:

    model_min = proper, live rows with  a + eps >= A*     + s + 2^-20
    model_max = rows               with  a + eps >= A_seed - 2 s - 2^-20,   count <= model_max + odd rows

with a = s dp, s = s_T s_q, A* the k-th class maximum of a - eps over all rows, A_seed the same over the seeding pass's
prefix.  The slack is rounding only: the device's class maxima and eps are directed-rounded f32 (each within ~1e-7 of
the model's, so within 2^-20), and its integer threshold floor((A - eps) / s) is computed through rounded reciprocals,
which moves it by less than one unit of s below the exact quotient.  A corpus in which A_seed == A* for every query
and no row lies within 2 units of its threshold pins the count exactly (test_exact_count).

Which kernel runs, its ring depth and the grids are restated from the source (scan_plan), and the case list is checked
to cover them on a machine without a GPU (test_plan_coverage).  CDB_TS_S8=1 forces the s8 form (monkeypatch)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from tests import prefilter_adversary as pa
from tests import prefilter_s8 as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "cosdata_b200", "csrc", "tensor_scan.cu")
SMS = 132            # H100 SXM: the SM count the plan coverage is stated for (the GPU tests read the device's own)
CHUNK = 2048         # queries per search chunk (search_device_locked)
CAP = 16384          # prefilter_k of every search here: no candidate list overflows (asserted against model_max)
TINY = 2.0 ** -20    # directed rounding of the device's class maxima and eps against the f64 model


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# ------------------------------------------------------------------ the plan, restated from csrc/tensor_scan.cu
def _source():
    with open(SRC) as f:
        return re.sub(r"//[^\n]*", "", f.read())


def _constexpr(src, name, defs=None):
    """value of a constexpr integer of tensor_scan.cu (its expression evaluated over the constants it names)"""
    defs = defs if defs is not None else dict(re.findall(r"constexpr\s+[\w:]+\s+(\w+)\s*=\s*([^;]+);", src))
    expr = " ".join(defs[name].replace("(size_t)", "").split())
    names = {v: _constexpr(src, v, defs) for v in re.findall(r"[A-Za-z_]\w*", expr)}
    return int(eval(expr, {"__builtins__": {}}, names))


def _num(src, pattern):
    m = re.search(pattern, src)
    assert m, f"{pattern!r} not found in csrc/tensor_scan.cu"
    return int(m.group(1))


def plan_constants():
    src = _source()
    c = {n: _constexpr(src, n) for n in ("TS8_MAX_STAGES", "TS8_MIN_STAGES", "TS8_KB_BYTES", "TS8_SMEM_FIXED", "TS_BLOCK_M",
                                         "TS_BLOCK_N", "TS8_HALF")}
    c["room_kb"] = _num(src, r"const size_t room = (\d+) \* 1024 - TS8_SMEM_FIXED;")
    c["k_resident"] = _num(src, r"a\.stages = k <= (\d+) && fit >= TS8_MIN_STAGES \? std::min\(fit, TS8_MAX_STAGES\) : 0;")
    c["seed_tiles"] = _num(src, r"seed_tiles = std::min<uint32_t>\(a\.ntiles, (\d+)\);")
    c["seed_after"] = _num(src, r"if \(a\.ntiles > (\d+)\) \{")
    c["seed_per_cta"] = _num(src, r"std::max<uint32_t>\(1, seed_tiles / (\d+)\)")
    c["main_per_cta"] = _num(src, r"std::max<uint64_t>\(1, total_tiles / (\d+)\)")
    enum = re.search(r"enum : int \{([^}]*)\}", src).group(1)
    c["prof_slots"] = [s.strip() for s in enum.split(",") if s.strip()]
    return c


PLAN = plan_constants()
SEED_ROWS = PLAN["seed_tiles"] * PLAN["TS_BLOCK_N"]


def s8_stages(dim, k):
    """tensor_scan_s8_device: the resident kernel's ring depth, 0 = the streamed tensor_scan_kernel runs"""
    kblocks = -(-dim // 128)
    slots = (PLAN["room_kb"] * 1024 - PLAN["TS8_SMEM_FIXED"]) // PLAN["TS8_KB_BYTES"]
    fit = slots - kblocks if slots > kblocks else 0
    return min(fit, PLAN["TS8_MAX_STAGES"]) if k <= PLAN["k_resident"] and fit >= PLAN["TS8_MIN_STAGES"] else 0


def scan_plan(n, nq, dim, k, sms=SMS):
    """run_tensor_scan for one chunk of nq <= 2048 queries: kernel, ring depth, NG, and per launch (seeding pass, main
    pass) its corpus tiles, CTAs per query tile G and the corpus tiles T of every CTA of a group"""
    assert nq <= CHUNK
    stages = s8_stages(dim, k)
    mtiles, ntiles = -(-nq // PLAN["TS_BLOCK_M"]), -(-n // PLAN["TS_BLOCK_N"])
    launches = []
    if ntiles > PLAN["seed_after"]:
        st = min(ntiles, PLAN["seed_tiles"])
        per_m = min(max(1, sms // mtiles), max(1, st // PLAN["seed_per_cta"]))
        launches.append(("seed", st, per_m))
    grid = min(sms, max(1, mtiles * ntiles // PLAN["main_per_cta"]))
    grid = max(1, grid // mtiles) * mtiles
    assert grid <= sms
    launches.append(("main", ntiles, grid // mtiles))
    out = []
    for name, nt, G in launches:
        T = [(nt - g + G - 1) // G if g < nt else 0 for g in range(G)]
        assert min(T) >= 2, (name, nt, G, T)      # the grids leave no CTA without a corpus tile, or with just one
        out.append({"launch": name, "ntiles": nt, "G": G, "T": T})
    return {"kernel": "resident" if stages else "streamed", "stages": stages, "ng": pa.ng_for_k(k), "mtiles": mtiles,
            "ntiles": ntiles, "kblocks": -(-dim // 128), "launches": out}


def chunk_sizes(nq):
    return [min(CHUNK, nq - o) for o in range(0, nq, CHUNK)]


def profiled_tiles(p):
    """TS_PROF_TILES of one chunk.  tensor_scan_s8_kernel: thread 0 of each consumer warpgroup adds the CTA's T (each
    warpgroup takes one half of each of the T tiles).  tensor_scan_kernel: thread 0 of each consumer warpgroup adds its
    tile counter t, which ends at the CTA's T (each warpgroup takes 64 queries of every whole tile).  So both count
    2 T per CTA, summed over mtiles CTAs per group and both launches."""
    return sum(2 * p["mtiles"] * sum(l["T"]) for l in p["launches"])


# ------------------------------------------------------------------ cases
# name: (dim, ks, n, nq, seed).  n mod 256 and nq are chosen so that together the cases cover every ring depth, both
# kernels, every NG, partial tiles and query tiles (test_plan_coverage lists what they cover)
CASES = {
    "d768_r6": (768, (10,), 256 * 65 + 128, 512, 11),
    "d300_r6_drift": (300, (10,), 256 * 64 + 1, 1040, 12),
    "d808_r5": (808, (1, 12), 256 * 66 + 127, 300, 13),
    "d1000_r4": (1000, (12,), 256 * 67 + 129, 130, 14),
    "d1100_streamed": (1100, (1, 10), 256 * 64 + 255, 100, 15),
    "d640_ng32": (640, (13, 28), 256 * 66, 512, 16),
    "d256_ng64_chunks": (256, (29, 64), 256 * 64 + 77, CHUNK + 300, 17),
}
EXACT_DIMS = (768, 808, 1000, 1100)     # test_exact_count: stages 6, 5, 4 and the streamed kernel
EXACT_N, EXACT_NQ, EXACT_K = 256 * 70 + 200, 160, 10
EDGE_DIMS = (808, 1000)                 # test_deleted_zero_and_odd_rows: stages 5 and 4, HAS_DEG
ADV_DIMS = (640, 808, 1000, 1100)       # one D per ring depth, and D > 1024


def covered():
    """(kernel, stages, NG) combinations, n mod 256, Ds and the CTA tile counts of the cases"""
    combos, mods, odd_dims, mtiles, resident_T = set(), set(), set(), set(), set()
    multi = False
    for dim, ks, n, nq, _ in CASES.values():
        mods.add(n % 256)
        multi |= nq > CHUNK
        for k in ks:
            for m in chunk_sizes(nq):
                p = scan_plan(n, m, dim, k)
                combos.add((p["kernel"], p["stages"], p["ng"]))
                mtiles.add(p["mtiles"])
                if dim % 128:
                    odd_dims.add((p["kernel"], p["stages"]))
                if p["kernel"] == "resident":
                    resident_T |= {t for l in p["launches"] for t in l["T"]}
    for dim in EXACT_DIMS + ADV_DIMS + EDGE_DIMS:
        p = scan_plan(EXACT_N, EXACT_NQ, dim, EXACT_K)
        combos.add((p["kernel"], p["stages"], p["ng"]))
    return combos, mods, odd_dims, mtiles, resident_T, multi


def test_plan_coverage():
    # the stage rule: 6 stages up to D = 768, 5 for 769..896, 4 for 897..1024, the streamed kernel above, and k > 12
    assert [s8_stages(d, 10) for d in (128, 640, 768, 769, 896, 897, 1024, 1025, 1100)] == [6, 6, 6, 5, 5, 4, 4, 0, 0]
    assert s8_stages(768, 12) == 6 and s8_stages(768, 13) == 0
    combos, mods, odd_dims, mtiles, resident_T, multi = covered()
    print("covered (kernel, stages, NG):", sorted(combos))
    assert combos >= {("resident", 6, 16), ("resident", 5, 16), ("resident", 4, 16), ("streamed", 0, 16),
                      ("streamed", 0, 32), ("streamed", 0, 64)}, combos
    assert {pa.ng_for_k(k) for c in CASES.values() for k in c[1]} == {16, 32, 64}
    assert {k for c in CASES.values() for k in c[1]} >= {1, 12, 13, 28, 29, 64}
    # D not a multiple of 128 at each ring depth and on the streamed kernel
    assert odd_dims >= {("resident", 6), ("resident", 5), ("resident", 4), ("streamed", 0)}, odd_dims
    assert mods >= {0, 1, 127, 128, 129, 255}, mods
    assert 1 in mtiles and max(mtiles) >= 9, mtiles          # one query tile; enough for the bounded-drift window
    assert any(nq % 128 for _, _, _, nq, _ in CASES.values()) and multi
    # a resident CTA with an odd number of corpus tiles, and one with the fewest the grids allow (2: seeding pass)
    assert any(t % 2 for t in resident_T) and min(resident_T) == 2, resident_T
    # the exact-count corpus: every ring depth and the streamed kernel, a partial last tile with rows in both halves
    assert sorted(s8_stages(d, EXACT_K) for d in EXACT_DIMS) == [0, 4, 5, 6] and EXACT_N % 256 > 128
    assert sorted(s8_stages(d, 10) for d in ADV_DIMS) == [0, 4, 5, 6]
    assert sorted(s8_stages(d, 10) for d in EDGE_DIMS) == [4, 5]


# ------------------------------------------------------------------ the model's bracket
def model_counts(x, q, k, deleted=None, has_deg=False, block=256):
    """-> (model_min, model_max, A_seed == A*) per query (model_max without the odd rows every list starts with)"""
    xh, ok = ps.normalized(x)
    live = ok if deleted is None else ok & ~deleted
    corpus = ps.quantize_corpus(x, deleted)
    lo, hi, same = [], [], []
    for b in range(0, len(q), block):
        dp, s, e = ps.filter_terms(q[b:b + block], x, corpus=corpus)
        a_all, a_seed = ps.filter_bounds(dp, s, e, k, has_deg, SEED_ROWS)
        up = dp * s + e
        lo.append(((up >= a_all[:, None] + s + TINY) & live[None, :]).sum(axis=1))
        hi.append((up >= a_seed[:, None] - 2 * s - TINY).sum(axis=1))
        same.append(a_seed == a_all)
    return np.concatenate(lo), np.concatenate(hi), np.concatenate(same)


def check_search(ix, x, q, k, s8=True, live=None, id_base=0, oracle_rows=16, **kw):
    """search q (candidate counts of the last chunk read right after it), then ids and score bits against exact_only and
    the CPU oracle over the live rows (first oracle_rows queries).  -> (counts of the last chunk, ids)"""
    st0 = ix.stats()
    ids, scores, _, _ = ix.batch_search(q, k, prefilter_k=CAP, **kw)
    counts = ix.last_candidate_counts(chunk_sizes(len(q))[-1])
    st1 = ix.stats()
    chunks = len(chunk_sizes(len(q)))
    assert st1["s8_searches"] - st0["s8_searches"] == (chunks if s8 else 0), (st0, st1)
    assert st1["tensor_searches"] - st0["tensor_searches"] == chunks and st1["fallbacks"] == st0["fallbacks"], (st0, st1)
    ids_e, scores_e, _, _ = ix.batch_search(q, k, exact_only=True)
    assert np.array_equal(ids, ids_e), np.argwhere(ids != ids_e)[:5]
    assert np.array_equal(bits(scores), bits(scores_e))
    rows = np.arange(len(x)) if live is None else live
    w_ids, w_scores = orc.brute_topk_f32(x[rows], q[:oracle_rows], k)
    assert np.array_equal(ids[:oracle_rows], rows[w_ids] + id_base)
    assert np.array_equal(bits(scores[:oracle_rows]), bits(w_scores))
    return counts, ids


def check_bracket(counts, x, q_last, k, deleted=None, has_deg=False, n_odd=0):
    lo, hi, _ = model_counts(x, q_last, k, deleted, has_deg)
    assert (hi + n_odd < CAP).all()                    # so no list overflowed: every emission was counted
    bad = np.flatnonzero((counts < lo) | (counts > hi + n_odd))
    assert not bad.size, [(int(i), int(lo[i]), int(counts[i]), int(hi[i]) + n_odd) for i in bad[:8]]
    return lo, hi


# ------------------------------------------------------------------ GPU
_INDEXES = {}


@pytest.fixture(scope="module")
def indexes():
    yield _INDEXES
    for ix, _, _ in _INDEXES.values():
        ix.close()
    _INDEXES.clear()


def case_index(indexes, name):
    if name not in indexes:
        dim, _, n, nq, seed = CASES[name]
        x, q = orc.synth_matrix(8000 + seed, n, dim), orc.synth_matrix(8100 + seed, nq, dim)
        ix = cdb.DenseIndex(dim=dim, capacity=n)
        ix.append(x)
        indexes[name] = (ix, x, q)
    return indexes[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_candidate_bracket(name, indexes, monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", "1")
    dim, ks, n, nq, _ = CASES[name]
    ix, x, q = case_index(indexes, name)
    q_last = q[len(q) - chunk_sizes(len(q))[-1]:]
    for k in ks:
        counts, _ = check_search(ix, x, q, k)
        check_bracket(counts, x, q_last, k)


def scan_profile(enable):
    """cdb_debug_scan_profile: switches the instrumented scan on / off, -> the TS_PROF_* sums since the previous call"""
    from cosdata_b200 import _lib
    fn = _lib.load().cdb_debug_scan_profile
    fn.argtypes, fn.restype = [C.c_int32, C.POINTER(C.c_uint64)], C.c_int32
    out = (C.c_uint64 * (len(PLAN["prof_slots"]) - 1))()
    assert fn(1 if enable else 0, out) == 0
    return dict(zip(PLAN["prof_slots"], [int(v) for v in out]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c for c in CASES if max(CASES[c][1]) <= 12])
def test_profiled_scan_counts_tiles(name, indexes, monkeypatch):
    import torch
    monkeypatch.setenv("CDB_TS_S8", "1")
    dim, ks, n, nq, _ = CASES[name]
    ix, x, q = case_index(indexes, name)
    k = max(ks)
    q = q[:CHUNK]
    p = scan_plan(n, len(q), dim, k, sms=torch.cuda.get_device_properties(0).multi_processor_count)
    ids0, scores0, _, _ = ix.batch_search(q, k, prefilter_k=CAP)
    counts0 = ix.last_candidate_counts(len(q))
    try:
        scan_profile(True)
        ids, scores, _, _ = ix.batch_search(q, k, prefilter_k=CAP)
        prof = scan_profile(False)
    finally:
        scan_profile(False)
    assert np.array_equal(ids, ids0) and np.array_equal(bits(scores), bits(scores0))
    assert prof["TS_PROF_TILES"] == profiled_tiles(p), (prof, p)
    assert prof["TS_PROF_CTAS"] == sum(p["mtiles"] * l["G"] for l in p["launches"]), (prof, p)
    assert (prof["TS_PROF_BOUND_ROUNDS"] > 0) == (p["kernel"] == "resident"), (prof, p)
    # the bound may rise at other moments than in the uninstrumented run, but stays within the model's bracket
    lo, hi, _ = model_counts(x, q, k)
    counts = ix.last_candidate_counts(len(q))
    assert ((counts >= lo) & (counts <= hi)).all() and ((counts0 >= lo) & (counts0 <= hi)).all()


# ------------------------------------------------------------------ exact count
def _unit_rows(rng, q_hat, cos):
    """rows with the given cosine to the unit queries q_hat: cos q_hat + sin u, u uniform and orthogonal to q_hat"""
    u = rng.uniform(-1, 1, q_hat.shape)
    u -= (u * q_hat).sum(axis=1, keepdims=True) * q_hat
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return (cos[:, None] * q_hat + np.sqrt(1 - cos ** 2)[:, None] * u).astype(np.float32)


def exact_count_data(dim, seed, n=EXACT_N, nq=EXACT_NQ, k=EXACT_K):
    """-> (x, q, model count per query) of a corpus on which the s8 filter's candidate count is fixed:
    * every query's top-k class maxima are set by rows in the seeding prefix (so A_seed == A*: every emission of the
      main pass uses the same bound, whatever the timing);
    * the partial last tile (both halves) holds rows built just above and just below the queries' thresholds;
    * no row's dp lies within 2 of its (query, tile) threshold (A* - eps) / s, so the device's rounding cannot move it."""
    ng = pa.ng_for_k(k)
    rng = np.random.default_rng(seed)
    x = orc.synth_matrix(9000 + seed, n, dim).copy()
    q = orc.synth_matrix(9100 + seed, nq, dim)
    q_hat = q.astype(np.float64) / np.linalg.norm(q.astype(np.float64), axis=1, keepdims=True)
    last = n - n % 256
    tail = np.arange(last, n)
    tq = (tail - last) % nq
    for it in range(30):
        dp, s, e = ps.filter_terms(q, x)
        lb = dp * s - e
        cm, arg = ps.class_maxima(lb, ng)
        top = np.take_along_axis(arg, np.argsort(-cm, axis=1)[:, :k], axis=1)
        need = np.unique(top)
        out = need[need >= SEED_ROWS]
        a_all, a_seed = ps.filter_bounds(dp, s, e, k, False, SEED_ROWS)
        if it == 0:
            # the last tile: rows for query tq at cosines around its threshold, where a + eps = A*
            frac = np.where((tail - last) % 4 < 2, -1.0, 1.0) * (0.15 + 0.2 * ((tail - last) // nq % 3))
            cos = a_all[tq] - e[tq, tail] + frac * e[tq, tail]
            x[tail] = _unit_rows(rng, q_hat[tq], np.clip(cos, -0.99, 0.99))
            continue
        if out.size:
            # move the class-argmax rows into the prefix (same class), then requantize
            taken = set(need.tolist())
            for r in out:
                free = [c for c in range(int(r % ng), SEED_ROWS, ng) if c not in taken]
                r2 = int(rng.choice(free))
                x[[r, r2]] = x[[r2, r]]
                taken.add(r2)
            continue
        t = (a_all[:, None] - e) / s
        near = np.abs(dp - t) <= 2
        if not near.any():
            break
        bad = np.unique(np.flatnonzero(near.any(axis=0)))
        assert not np.isin(bad, need).any(), "a row that sets a class maximum lies at another query's threshold"
        for r in bad:           # a fresh row: uniform, or (last tile) another near-threshold row of its query
            if r >= last:
                j = (r - last) % nq
                x[r] = _unit_rows(rng, q_hat[j:j + 1], np.clip([a_all[j] - e[j, r] + 0.5 * e[j, r]], -0.99, 0.99))[0]
            else:
                x[r] = rng.uniform(-1, 1, dim).astype(np.float32)
    else:
        raise AssertionError("no exact-count corpus found")
    # the fixture's preconditions
    assert (a_seed == a_all).all()
    assert not (np.abs(dp - (a_all[:, None] - e) / s) <= 2).any()
    emit = dp >= (a_all[:, None] - e) / s
    assert emit[:, last:last + 128].any() and emit[:, last + 128:].any()          # emissions in both halves
    below = ~emit[:, last:] & (dp[:, last:] * s[:, last:] + 2 * e[:, last:] >= a_all[:, None])
    assert below[:, :128].any() and below[:, 128:].any()                          # and rows just below the threshold
    return x, q, emit.sum(axis=1)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", EXACT_DIMS)
def test_exact_count(dim, monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", "1")
    x, q, want = exact_count_data(dim, seed=dim)
    p = scan_plan(len(x), len(q), dim, EXACT_K)
    ix = cdb.DenseIndex(dim=dim, capacity=len(x))
    ix.append(x)
    counts, _ = check_search(ix, x, q, EXACT_K)
    ix.close()
    print(f"exact count D={dim} ({p['kernel']}, stages {p['stages']}): model {int(want.sum())} measured {int(counts.sum())}")
    bad = np.flatnonzero(counts != want)
    assert not bad.size, [(int(i), int(want[i]), int(counts[i])) for i in bad[:8]]


# ------------------------------------------------------------------ edges of the data (HAS_DEG)
@pytest.mark.gpu
@pytest.mark.parametrize("dim", EDGE_DIMS)
def test_deleted_zero_and_odd_rows(dim, monkeypatch):
    monkeypatch.setenv("CDB_TS_S8", "1")
    n, nq = 256 * 66 + 200, 260                     # last tile: a full lower half, 72 rows in the upper half
    last = 256 * 66
    x = orc.synth_matrix(9300 + dim, n, dim).copy()
    q = orc.synth_matrix(9301 + dim, nq, dim)
    x[10 * 256:11 * 256] = 0.0                      # a tile of zero rows: s_T = 0
    odd = np.array([77, 5000, 9999, last + 3, last + 140])
    x[odd] = 1e-25                                  # odd degenerate rows: on every candidate list
    dead = np.concatenate([np.arange(20 * 256, 21 * 256), [last + 130, last + 150, n - 1]])   # a whole tile, upper half
    id_base = 2 ** 32 - 1 - n                       # warpgroup 1's ids in the last tile reach the top of the id range
    deleted = np.zeros(n, bool)
    deleted[dead] = True
    ix = cdb.DenseIndex(dim=dim, capacity=n, id_base=id_base)
    ix.append(x)
    assert (ix.delete_rows(dead) == 0).all()
    st = ix.stats()
    assert st["zero_rows"] == 256 and st["odd_rows"] == len(odd)
    assert s8_stages(dim, 10) in (4, 5)
    live = np.flatnonzero(~deleted)
    for k in (1, 10):
        counts, ids = check_search(ix, x, q, k, live=live, id_base=id_base, tensor_with_deleted=True)
        assert not np.isin(ids, dead + id_base).any()
        check_bracket(counts, x, q, k, deleted, has_deg=True, n_odd=len(odd))
    ix.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dim", ADV_DIMS)
def test_adversarial_corpus(dim, monkeypatch):
    # a filter at eps/2 loses the true top-k on this corpus (tests/prefilter_s8.py)
    monkeypatch.setenv("CDB_TS_S8", "1")
    n, k = 16384 + 300, 10
    x, q, nb = ps.adversarial_corpus(n, dim, 256, seed=dim)
    ix = cdb.DenseIndex(dim=dim, capacity=n)
    ix.append(x)
    counts, ids = check_search(ix, x, q, k)
    b0 = (np.arange(len(q)) % nb) * ps.TILE
    assert ((ids > b0[:, None]) & (ids <= b0[:, None] + 64)).all()
    check_bracket(counts, x, q, k)
    ix.close()


# ------------------------------------------------------------------ the gate (no CDB_TS_S8)
@pytest.mark.gpu
def test_gate_boundaries(monkeypatch):
    monkeypatch.delenv("CDB_TS_S8", raising=False)
    n = 16384 + 50
    for dim, nq, s8 in ((256, 511, False), (256, 512, True), (255, 512, False)):
        x, q = orc.synth_matrix(9400 + dim, n, dim), orc.synth_matrix(9401 + nq, nq, dim)
        ix = cdb.DenseIndex(dim=dim, capacity=n)
        ix.append(x)
        check_search(ix, x, q, 10, s8=s8)
        ix.close()
