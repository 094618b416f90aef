"""The HNSW warp traversal (hw_traverse_level, hnsw_traverse.cuh) at its queue, fixed-set and metadata limits, exact against
the oracles: ids, score bits, counts, error flags, evaluation and pop counts, and graphs array for array.

  1. every pool class of ef (EFP 128 .. 4096) on a 64-regular graph, the pool trims (EFP 512, 1024) and the exact
     selection (EFP 128) proven by the profile counters, a pool that runs dry, and u8 / 1-bit rows whose tied scores leave the order to the ids;
  2. crafted adjacency at non-power-of-two neighbour counts: duplicates, aliasing ids in either half of a pop and across the
     halves (the slot-order `resolve` branch), empty slots, self links and links to the entry;
  3. the graph writers at large ef_construction and neighbour counts 20 / 48;
  4. metadata widths 8 .. 4096 with schema-like dimension vectors, the filter compared beyond one warp's width;
  5. the metadata cosine exactly at the 0.99 threshold and just above it;
  6. 1 .. 4096 filter rows per query, and 4097 refused by the host form, flagged per query by the device form;
  7. the metadata form's shared-memory carve restated, one step on each side of 200 KB;
  8. the replica writers at 33 and 257 metadata dims.

The fixed set (PerformantFixedSet, fixedset.rs) has nb buckets of 64 bits and hashes an id to bucket (id >> 6) & (nb - 1),
bit id & 63, so a traversal scores at most 64 * nb nodes.  With nb = 64 that is 4096 <= 2 * EFP - 64 + (pops so far) for
EFP >= 2048: the pool can never fill there, and its trims are reachable only at EFP 512 and 1024 (asserted below)."""
import functools
from itertools import combinations

import numpy as np
import pytest

import cosdata_b200 as cdb
import oracle as orc
from oracle import pyhnsw, pymeta
from tests import mdgraph, pydelete, pydelete_md, pyinsert

ST, MK = cdb.StorageType, cdb.DistanceMetricKind
EMPTY = 0xFFFFFFFF
ROOT_ID, QUERY_ID = 0xFFFFFFFF, 0xFFFFFFFE
BAD_FILTER = 8
gpu = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def efp(ef):   # hn_efp: the padded pool size
    return max(128, 1 << max(0, (ef - 1).bit_length()))


def fs_bit(i, nb):   # PerformantFixedSet bucket and bit of id i as one bit index
    return (((int(i) >> 6) & (nb - 1)) << 6) | (int(i) & 63)


# ----------------------------------------------------------------------------- 7 (CPU). the carve, restated
def round_up(x, m):
    return (x + m - 1) // m * m


def carve(pitch, ef, md=False, M=0):
    """hw_carve(pitch, ef, md, M).total: the warp's dynamic shared memory in bytes"""
    p = efp(ef)
    stage_pitch = round_up(pitch, 16) + 16
    stage_rows = min(32, max(1, 18700 // stage_pitch))
    o = round_up(pitch, 16)                        # the query's code
    o += 2 * p * 8 + p * 8 + 64 * 8 + 8            # qkeys, rkeys, nkeys, mbarrier
    o += 128 * 4                                   # the fixed set
    o += 2 * p * 4 + p * 4 + 64 * 4 + 64 * 4       # qnodes, rnodes, nnodes, nrow
    if md:
        o = round_up(o, 8)
        o += 256 * 8 + 256 * 4 + 4 * 4 + M * 4     # z keys, z nodes, {f0, f1, count}, the filter's dims as i32
    return round_up(o, 16) + stage_rows * stage_pitch


LIMIT = 200 * 1024
CARVE_D, CARVE_EF = 6144, 4096                    # f32 rows of 24 KB, pool class 4096


def carve_edge():
    """(M accepted, M + 1 refused) at f32 x CARVE_D, ef CARVE_EF"""
    pitch = 4 * CARVE_D
    m = max(M for M in range(1, 4097) if carve(pitch, CARVE_EF, True, M) <= LIMIT)
    return m, m + 1


def test_carve_restatement_straddles_200kb():
    from tests.test_gpu_hnsw_rowsize import carve_bytes
    for pitch in (16, 32, 48, 1536, 1552, 3072, 8192, 16384, 24576):
        for ef in (1, 128, 129, 512, 1000, 4096):
            assert carve(pitch, ef) == carve_bytes(pitch, ef), (pitch, ef)
            # the metadata form adds the z list, three counters and M i32 dims, rounded to 16 with the rest
            assert carve(pitch, ef, True, 0) - carve(pitch, ef) in range(3088, 3088 + 32)
    ok, bad = carve_edge()
    pitch = 4 * CARVE_D
    assert carve(pitch, CARVE_EF, True, ok) <= LIMIT < carve(pitch, CARVE_EF, True, bad)
    assert 0 < ok < 4096 and carve(pitch, CARVE_EF) <= LIMIT
    # at small D no metadata width reaches the limit: the refusal needs wide rows
    assert carve(32, 4096, True, 4096) < LIMIT


# ----------------------------------------------------------------------------- helpers: plain graphs
def plain_index(stored, st, metric, levels, nb, nb0, entry, node_row, adj, child):
    """stored: data rows + the root row (last); -> (index, FlatGraph over the index's own codes)"""
    n1, dim = stored.shape
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n1, keep_raw_f32=True)
    ix.append(stored)
    ix.set_graph(levels, nb, nb0, entry, n1 - 1, node_row, adj, child)
    codes, mags = ix.read_codes(0, n1)
    fg = pyhnsw.FlatGraph(int(metric), int(st), dim, codes, mags, n1 - 1, levels, nb, nb0, entry, node_row, adj, child)
    return ix, fg


def gpu_search(ix, queries, k, ef, shortlist=64):
    ev0, pp0 = ix.hnsw_counters()
    ids, scores, counts, err = ix.batch_search(queries, k, cdb.SearchMode.HNSW, ef_search=ef, shortlist_size=shortlist)
    ev1, pp1 = ix.hnsw_counters()
    return ids, scores, counts, err, ev1 - ev0, pp1 - pp0


def assert_search_equal(got, want, what):
    assert np.array_equal(got[3], want[3]), what
    assert np.array_equal(got[2], want[2]), what
    assert np.array_equal(got[0], want[0]), what
    assert np.array_equal(bits(got[1]), bits(want[1])), what
    assert (got[4], got[5]) == (want[4], want[5]), what


def one_level(adj, n1):
    return [np.arange(n1, dtype=np.uint32)], [np.ascontiguousarray(adj, np.uint32).ravel()], [np.zeros(n1, np.uint32)]


# ----------------------------------------------------------------------------- 1. pool and ef classes
EFS = (1, 2, 127, 128, 129, 511, 512, 513, 1024, 2047, 2048, 4095, 4096)


@functools.lru_cache(maxsize=None)
def regular_graph(n=20000, dim=16, nb0=64, seed=41):
    """n rows + root, each node linking 64 random nodes on level 0 only: every early pop brings up to 64 fresh candidates"""
    rng = np.random.default_rng(seed)
    stored = rng.uniform(-0.9, 0.9, size=(n + 1, dim)).astype(np.float32)
    adj = rng.integers(0, n + 1, size=(n + 1, nb0)).astype(np.uint32)
    return stored, adj


@gpu
def test_every_pool_class_equals_oracle_and_trims_where_the_pool_can_fill():
    # seeds: graph 41, queries 42 (32 queries below ef 1024, 12 above).  On an H100 they gave, per pool class, (trims, exact
    # selections): 128 (2397, 8), 256 (468, 0), 512 (673, 0), 1024 (140, 0), 2048 and 4096 (0, 0).  Above EFP 128 the window
    # of usable pivot ranks, [R, 2 * EFP - 96] of about 2 * EFP - 64 entries, is about half the pool, so the 12 sampled
    # pivots practically never all miss it and the exact selection stays a fallback of the small classes.
    stored, adj = regular_graph()
    n1, nb0 = stored.shape[0], adj.shape[1]
    ix, fg = plain_index(stored, ST.HalfPrecisionFP, MK.Cosine, 0, nb0, nb0, 17, *one_level(adj, n1))
    rng = np.random.default_rng(42)
    k, prof = 10, {}
    for ef in EFS:
        nq = 32 if ef < 1024 else 12
        queries = rng.uniform(-0.9, 0.9, size=(nq, stored.shape[1])).astype(np.float32)
        want = pyhnsw.search_batch(fg, stored[:-1], queries, k, ef_search=ef)
        assert (want[3] == 0).all() and (want[2] > 0).all(), ef
        if ef <= 1024:
            assert want[5] == nq * ef, ef                        # every traversal runs its ef pops
        assert_search_equal(gpu_search(ix, queries, k, ef), want, ef)
        ix.hnsw_profile(enable=True, read=False)                 # the instrumented kernel walks the same path
        assert_search_equal(gpu_search(ix, queries, k, ef), want, ("profiled", ef))
        p = ix.hnsw_profile(enable=False, read=True)
        assert p["pops"] == want[5], ef
        prof.setdefault(efp(ef), []).append((ef, p["trims"], p["exact_selections"]))
    summary = {c: (sum(t for _, t, _ in v), sum(e for _, _, e in v)) for c, v in prof.items()}
    print("pool class -> (trims, exact selections):", summary)
    for c in (512, 1024):
        assert summary[c][0] > 0, (c, prof[c])
    for c in (2048, 4096):                                       # 64 * nb0 scored nodes at most: the pool never fills
        assert summary[c][0] == 0, (c, prof[c])
    assert summary[128][1] > 0, prof[128]
    ix.close()


@gpu
def test_pool_runs_dry_before_ef_pops():
    # a 300-node component holding the entry, and the rest of the graph unreachable from it: ef 4096 pops all 300 and stops
    n, small, dim, nb0 = 3000, 300, 16, 64
    rng = np.random.default_rng(7)
    stored = rng.uniform(-0.9, 0.9, size=(n + 1, dim)).astype(np.float32)
    adj = np.empty((n + 1, nb0), np.uint32)
    adj[:small] = rng.integers(0, small, size=(small, nb0))
    adj[small:] = rng.integers(small, n + 1, size=(n + 1 - small, nb0))
    adj[rng.random(adj.shape) < 0.2] = EMPTY
    ix, fg = plain_index(stored, ST.HalfPrecisionFP, MK.Cosine, 0, nb0, nb0, 5, *one_level(adj, n + 1))
    queries = rng.uniform(-0.9, 0.9, size=(6, dim)).astype(np.float32)
    for ef in (300, 301, 4096):
        want = pyhnsw.search_batch(fg, stored[:-1], queries, 10, ef_search=ef)
        assert want[5] == 6 * small and want[4] == 6 * small, ef  # every node of the component scored and popped once
        assert_search_equal(gpu_search(ix, queries, 10, ef), want, ef)
        ids = gpu_search(ix, queries, 10, ef)[0]
        assert (ids < small).all()
    ix.close()


@gpu
@pytest.mark.parametrize("st,metric,dim", [(ST.UnsignedByte, MK.Cosine, 3), (ST.SubByte1, MK.DotProduct, 8)])
def test_tied_scores_leave_the_order_to_the_ids(st, metric, dim):
    n, nb0 = 6000, 32
    rng = np.random.default_rng(int(st) + 3)
    stored = rng.choice(np.float32([-0.5, 0.5]), size=(n + 1, dim))   # 8 / 256 distinct rows: codes and raw scores tie
    adj = rng.integers(0, n + 1, size=(n + 1, nb0)).astype(np.uint32)
    ix, fg = plain_index(stored, st, metric, 0, nb0, nb0, 0, *one_level(adj, n + 1))
    codes = fg.codes[:n]
    assert np.unique(codes, axis=0).shape[0] < n // 4            # most rows share their code with others
    queries = rng.uniform(-0.9, 0.9, size=(16, dim)).astype(np.float32)
    for ef in (64, 513, 2048):
        want = pyhnsw.search_batch(fg, stored[:-1], queries, 20, ef_search=ef)
        assert_search_equal(gpu_search(ix, queries, 20, ef), want, ef)
        ok = want[3] == 0
        assert ok.any(), ef
        assert (np.diff(want[1][ok], axis=1) == 0).any(), ef     # tied scores inside the results: ordered by id
    ix.close()


# ----------------------------------------------------------------------------- 2. fixed set and adjacency
N_ROWS = 9000   # data rows; the root is row N_ROWS.  Ids reach past 4096 = 64 * 64, so ids alias at every neighbour count


def alias_hole(i, nb):
    """another id on the same fixed-set bit: flip the lowest bucket bit outside the mask (a hole of a non-power-of-two
    mask), or bit 12 when the mask has none"""
    mask = nb - 1
    hole = next((b for b in range(6) if not (mask >> b) & 1), None)
    return i ^ (1 << (6 + hole)) if hole is not None else i ^ 4096


def crafted_ids(self_rows, nb, entry_row, rng):
    """[cnt, nb] neighbour rows: random rows and empty slots, with fixed slot patterns laid over them:
       0,1: an id and its alias (same bit, lower half)    2,3: one id twice    4: EMPTY    5: the node itself    6: the entry
       7,31: an id and its bit-12 alias (lower half)      12,32: an id and its alias across the halves
       34,50: an id and its bit-12 alias (upper half)     40,63: one id twice (upper half)"""
    cnt = self_rows.size
    ids = rng.integers(0, N_ROWS + 1, size=(cnt, nb)).astype(np.int64)
    ids[rng.random((cnt, nb)) < 0.1] = EMPTY
    low = lambda: rng.integers(0, 4096, cnt)
    a, c, f, g = low(), low(), low(), low()
    d, h = rng.integers(0, N_ROWS, cnt), rng.integers(0, N_ROWS, cnt)
    plan = {0: a, 1: alias_hole(a, nb), 2: d, 3: d, 4: EMPTY, 5: self_rows, 6: entry_row, 7: c, 31: c ^ 4096,
            12: f, 32: alias_hole(f, nb), 34: g, 50: g ^ 4096, 40: h, 63: h}
    for pos, v in plan.items():
        if pos < nb:
            ids[:, pos] = v
    return ids


def row_id(r):
    return ROOT_ID if r == N_ROWS else int(r)


def resolve_kinds(slot_rows, take, nb, seeded):
    """the pairs of one pop that reach the slot-order `resolve` branch: two slots whose bit is clear when the pop starts and
    that share it -> {"lower", "upper", "across"}"""
    cand = [(s, fs_bit(row_id(r), nb)) for s, r in enumerate(slot_rows[:take]) if r != EMPTY]
    cand = [(s, b) for s, b in cand if b not in seeded]
    kinds = set()
    for (s1, b1), (s2, b2) in combinations(cand, 2):
        if b1 == b2:
            kinds.add("lower" if s2 < 32 else "upper" if s1 >= 32 else "across")
    return kinds


def expected_kinds(take, nb):
    want = set()
    if min(take, nb) >= 2:
        want.add("lower")
    if min(take, nb) >= 33:
        want.add("across")
    if min(take, nb) >= 51:
        want.add("upper")
    return want


NB_PAIRS = [(1, 64), (3, 63), (20, 48), (33, 33), (48, 20), (63, 3), (64, 1)]
SHORTLISTS = (1, 5, 32, 33, 64)


@gpu
@pytest.mark.parametrize("nb,nb0", NB_PAIRS, ids=[f"nb{a}-nb0{b}" for a, b in NB_PAIRS])
def test_crafted_adjacency_at_odd_neighbour_counts(nb, nb0):
    """Two levels over 9001 rows: level 1 holds every row in a shuffled order (node index != row), level 0 is the identity.
    Every adjacency list carries the slot patterns of crafted_ids, so each pop meets them; the first pop of each level is
    checked in Python to reach `resolve` for the pattern kinds its `take` covers (lower half from take 2, across the halves
    from 33, upper half from 51)."""
    dim = 16
    rng = np.random.default_rng(nb * 100 + nb0)
    stored = rng.uniform(-0.9, 0.9, size=(N_ROWS + 1, dim)).astype(np.float32)
    perm = rng.permutation(N_ROWS + 1).astype(np.uint32)           # level 1: node i is row perm[i]
    inv = np.empty_like(perm)
    inv[perm] = np.arange(perm.size, dtype=np.uint32)
    rows1 = crafted_ids(perm.astype(np.int64), nb, N_ROWS, rng)
    # the entry's own pairs on bits that the query and the entry do not hold: its first pop reaches `resolve` for sure
    for pos, v in ((0, 5), (1, alias_hole(5, nb)), (12, 6), (32, alias_hole(6, nb)), (34, 7), (50, 7 ^ 4096)):
        if pos < nb:
            rows1[inv[N_ROWS], pos] = v
    rows0 = crafted_ids(np.arange(N_ROWS + 1), nb0, N_ROWS, rng)
    adj1 = np.where(rows1 == EMPTY, EMPTY, inv[np.where(rows1 == EMPTY, 0, rows1)]).astype(np.uint32)
    adj0 = rows0.astype(np.uint32)
    entry = int(inv[N_ROWS])
    node_row = [np.arange(N_ROWS + 1, dtype=np.uint32), perm]
    ix, fg = plain_index(stored, ST.HalfPrecisionFP, MK.Cosine, 1, nb, nb0, entry, node_row, [adj0.ravel(), adj1.ravel()],
                         [np.zeros(N_ROWS + 1, np.uint32), perm])
    queries = rng.uniform(-0.9, 0.9, size=(24, dim)).astype(np.float32)
    qcodes, qmags = orc.quantize_batch(int(ST.HalfPrecisionFP), queries)
    k, ef = 10, 100
    reached = {}
    for sl in SHORTLISTS:
        want = pyhnsw.search_batch(fg, stored[:-1], queries, k, ef_search=ef, shortlist_size=sl)
        assert_search_equal(gpu_search(ix, queries, k, ef, sl), want, sl)
        assert (want[3] == 0).all()
        # the first pop of level 1 (the entry, the root) and of level 0 (the best level-1 result) of every query
        t1, t0 = min(sl, nb, 64), min(sl, nb0, 64)
        kinds1 = resolve_kinds(rows1[entry], t1, nb, {fs_bit(QUERY_ID, nb), fs_bit(ROOT_ID, nb)})
        kinds0 = set()
        for i in range(len(queries)):
            rc, rows, _, _, _ = pyhnsw.ann_search(fg, qcodes[i], qmags[i], ef_search=ef, shortlist_size=sl)
            e0 = int(rows[0])
            kinds0 |= resolve_kinds(rows0[e0], t0, nb0, {fs_bit(QUERY_ID, nb0), fs_bit(row_id(e0), nb0)})
        assert expected_kinds(t1, nb) <= kinds1, (sl, kinds1)
        assert expected_kinds(t0, nb0) <= kinds0, (sl, kinds0)
        reached[sl] = (sorted(kinds1), sorted(kinds0))
    print(f"nb {nb} / nb0 {nb0}: shortlist -> resolve kinds on the first pop of (level 1, level 0):", reached)
    ix.close()


# ----------------------------------------------------------------------------- 3. writers at large ef_construction
W_LEVELS, W_NB, W_NB0 = 3, 20, 48


def clustered(n, dim, seed):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(16, dim)).astype(np.float32)
    v = (centres[rng.integers(0, 16, n)] + 0.35 * rng.normal(size=(n, dim))).astype(np.float32)
    return (v / (np.abs(v).max() * 1.01)).astype(np.float32)


def assert_graph_equal(ix, e, metric):
    g, sc = ix.read_graph(), ix.read_graph_slot_scores()
    assert g["entry"] == e["entry"] and g["root_row"] == e["root_row"]
    for lv in range(g["num_levels"] + 1):
        assert np.array_equal(g["node_row"][lv], e["node_row"][lv]), lv
        assert np.array_equal(g["adj"][lv], e["adj"][lv]), lv
        if lv:
            assert np.array_equal(g["child"][lv], e["child"][lv]), lv
        assert np.array_equal(bits(sc[lv]), bits(pyinsert.slot_scores(metric, e["simkey"][lv], e["adj"][lv]))), lv


@gpu
@pytest.mark.parametrize("efc", [1, 129, 513, 1024])
def test_sequential_build_at_large_ef_construction(efc):
    st, metric, dim, n, seed = ST.HalfPrecisionFP, MK.Cosine, 16, 1200, 5
    vecs = clustered(n, dim, 11)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 1, keep_raw_f32=True)
    ix.append(vecs)
    ix.build_graph(W_LEVELS, W_NB, W_NB0, efc, 64, 1, seed)
    codes, mags = ix.read_codes(0, n + 1)
    o = pyinsert.Graph.init(int(metric), int(st), dim, codes, mags, n, W_LEVELS, W_NB, W_NB0)
    assert o.insert(0, n, ef_construction=efc, seed=seed).sum() == 0
    assert_graph_equal(ix, o.export(), int(metric))
    o.close()
    ix.close()


@gpu
def test_sequential_insert_and_delete_at_ef_construction_1024():
    st, metric, dim, n0, efc, seed = ST.HalfPrecisionFP, MK.Cosine, 16, 900, 1024, 7
    vecs = clustered(n0 + 150, dim, 13)
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n0 + 151, keep_raw_f32=True)
    ix.append(vecs[:n0])
    ix.build_graph(W_LEVELS, W_NB, W_NB0, efc, 64, 1, seed)
    ix.append(vecs[n0:])
    failed = ix.insert_graph(efc, 64, 1, seed)
    assert failed.size == 150 and failed.sum() == 0
    codes, mags = ix.read_codes(0, n0 + 151)
    o = pydelete.Graph.init(int(metric), int(st), dim, codes, mags, n0, W_LEVELS, W_NB, W_NB0)
    o.insert(0, n0, ef_construction=efc, seed=seed)
    o.insert(n0 + 1, 150, ef_construction=efc, seed=seed)
    assert_graph_equal(ix, o.export(), int(metric))
    rows = np.random.default_rng(3).choice(np.r_[0:n0, n0 + 1:n0 + 151], 40, replace=False).astype(np.uint32)
    rows = np.concatenate([rows, rows[:2]])                             # deleted twice: status 1
    status = ix.delete_rows(rows, 64, 1)
    assert np.array_equal(status, o.delete(rows)) and (status[-2:] == 1).all()
    assert_graph_equal(ix, o.export(), int(metric))
    ix.close()
    o.close()


# ----------------------------------------------------------------------------- helpers: graphs with metadata
def md_index(vecs, mg, st, metric):
    fg = mg.fg
    ix = cdb.DenseIndex(dim=vecs.shape[1], storage_type=st, metric=metric, capacity=vecs.shape[0], keep_raw_f32=True)
    ix.append(vecs)
    ix.set_graph(fg.num_levels, fg.neighbors_count, fg.level0_neighbors_count, fg.entry, fg.n, fg.node_row, fg.adj, fg.child)
    ix.set_graph_metadata(mg.md_bits, mg.md_mags, mg.node_id, mg.node_md, mg.pseudo_entry)
    return ix


def assert_filtered_equal(ix, mg, vecs, q, filters, k, ef):
    """host form == oracle (arrays; evaluation and pop counts over the error-free queries) -> the host result"""
    got = ix.batch_search_filtered(q, filters, k, ef_search=ef, shortlist_size=64)
    want = pymeta.search_batch_md(mg, vecs, q, filters, k, ef_search=ef, shortlist_size=64)
    assert np.array_equal(got[3], want[3])
    assert np.array_equal(got[2], want[2])
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(bits(got[1]), bits(want[1]))
    sel = np.flatnonzero(want[3] == 0)
    sub = [filters[i] for i in sel]
    e0 = ix.hnsw_counters()
    ix.batch_search_filtered(q[sel], sub, k, ef_search=ef, shortlist_size=64)
    e1 = ix.hnsw_counters()
    w = pymeta.search_batch_md(mg, vecs, q[sel], sub, k, ef_search=ef, shortlist_size=64)
    assert (e1[0] - e0[0], e1[1] - e0[1]) == (w[4], w[5])
    return got, want


def device_search(ix, q, filters, k, ef):
    import torch
    from tests.test_gpu_filtered_device import DeviceBatch
    b = DeviceBatch(ix, q, filters, k)
    s = torch.cuda.Stream()
    b.run(ix, s, ef_search=ef, shortlist_size=64)
    s.synchronize()
    return b.result()


def assert_same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8))


def pair_md(st, dim, M, qcode, qmag, filt, node_code, node_mag, node_id, node_bits):
    """calculate(x, y) on the GPU and in the oracle for one query side (no id, filter dims) per node side"""
    n = len(node_bits)
    fm = pymeta.query_filter_mag(filt)
    nm = np.array([pymeta.metadata_mag(b) for b in node_bits], np.float32)
    x = dict(codes=np.repeat(qcode[None], n, 0), mags=np.full(n, qmag, np.float32), ids=np.zeros(n, np.uint32),
             has_id=np.zeros(n, np.uint8), md_bits=np.repeat(np.asarray(filt, np.int32)[None], n, 0),
             md_mags=np.full(n, fm, np.float32), has_md=np.ones(n, np.uint8))
    y = dict(codes=np.repeat(node_code[None], n, 0), mags=np.full(n, node_mag, np.float32),
             ids=np.full(n, node_id, np.uint32), has_id=np.ones(n, np.uint8), md_bits=np.asarray(node_bits, np.int32),
             md_mags=nm, has_md=np.ones(n, np.uint8))
    val, status = cdb.DistanceMetric(MK.Cosine).calculate_pairs_md(st, dim, M, x, y)
    for i in range(n):
        vx = pymeta.VectorData(qcode, qmag, None, filt, fm)
        vy = pymeta.VectorData(node_code, node_mag, node_id, node_bits[i], nm[i])
        rc, w = pymeta.distance_md(int(MK.Cosine), int(st), dim, M, vx, vy)
        assert status[i] == rc and (rc or bits(val[i]) == bits(w)), i
    return val, status


# ----------------------------------------------------------------------------- 4. metadata width
WIDTHS = (8, 9, 16, 31, 32, 33, 64, 257, 1024, 4096)
MD_TYPES = [(ST.HalfPrecisionFP, "f16"), (ST.BFloat16, "bf16"), (ST.FullPrecisionFP, "f32")]


def flipped(pattern, d):
    f = np.asarray(pattern, np.int8).copy()
    f[d] ^= 1
    return f


@gpu
@pytest.mark.parametrize("st", [t for t, _ in MD_TYPES], ids=[s for _, s in MD_TYPES])
@pytest.mark.parametrize("M", WIDTHS)
def test_filtered_search_at_metadata_width(M, st):
    dim, k, ef = 16, 10, 64
    vecs, mg = mdgraph.build(n=300, dim=dim, md_dims=M, levels=3, nb=8, nb0=16, storage_type=int(st), metric=int(MK.Cosine),
                             seed=M, patterns=mdgraph.schema_patterns)
    q, filters = mdgraph.make_queries(vecs, mg, 40, seed=M + 1)
    # a pseudo node's pattern, exact and differing in one dim: 32 (past one warp), 33 and M - 1 -> (Pseudo, Metadata) arm
    # gives 1.0 for the exact pattern and -1.0 for every flip
    ps = int(np.flatnonzero((mg.node_id[0] > mdgraph.PSEUDO_ROOT_ID) & (mg.node_id[0] <= 0xFFFFFFFF - 2))[0])
    pat = mg.md_bits[mg.node_md[0][ps]]
    edge = [pat.astype(np.int8)] + [flipped(pat, d) for d in (32, 33, M - 1) if d < M]
    for i, f in enumerate(edge):
        filters[1 + 4 * i] = [f]
    filters[2] = edge
    ix = md_index(vecs, mg, st, MK.Cosine)
    got, _ = assert_filtered_equal(ix, mg, vecs, q, filters, k, ef)
    assert_same(device_search(ix, q, filters, k, ef), got)
    # the same arm pairwise
    codes, mags = orc.quantize_batch(int(st), np.concatenate([q[:1], vecs[-1:]]))
    for f, want in zip(edge, [1.0] + [-1.0] * (len(edge) - 1)):
        val, status = pair_md(st, dim, M, codes[0], mags[0], f, codes[1], mags[1], int(mg.node_id[0][ps]), [pat])
        assert status[0] == 0 and val[0] == want
    ix.close()


# ----------------------------------------------------------------------------- 5. the 0.99 threshold
def threshold_patterns(M):
    """(filter F, A: as many ones as F, all but ones/100 of them shared -> cosine exactly 0.99f, B: ones contained in F,
    1 % fewer -> cosine sqrt(0.99) = 0.99499)"""
    ones = 100 if M < 4096 else 400
    lost = ones // 100
    F = np.zeros(M, np.int32)
    F[:ones] = 1
    A = np.zeros(M, np.int32)
    A[lost:ones + lost] = 1
    B = np.zeros(M, np.int32)
    B[:ones - lost] = 1
    return F, A, B


@gpu
@pytest.mark.parametrize("M", [128, 4096])
def test_metadata_cosine_at_the_099_threshold(M):
    F, A, B = threshold_patterns(M)
    mag = lambda r: np.float32(pymeta.metadata_mag(r))
    assert np.float32(np.float32((F * A).sum()) / np.float32(mag(F) * mag(A))) == np.float32(0.99)
    assert np.float32(np.float32((F * B).sum()) / np.float32(mag(F) * mag(B))) > np.float32(0.99)
    st, dim, k, ef = ST.HalfPrecisionFP, 16, 10, 256

    def patterns(md_dims, n_patterns, rng):
        rest = mdgraph.schema_patterns(md_dims, n_patterns - 2, rng)
        return np.concatenate([A[None], B[None], rest])
    vecs, mg = mdgraph.build(n=400, dim=dim, md_dims=M, levels=3, nb=8, nb0=16, storage_type=int(st), metric=int(MK.Cosine),
                             seed=99, patterns=patterns)
    assert np.array_equal(mg.md_bits[2], A) and np.array_equal(mg.md_bits[3], B)
    # pairwise: a Metadata node with A is a strong mismatch, one with B takes the vector arm
    codes, mags = orc.quantize_batch(int(st), vecs[:2])
    val, status = pair_md(st, dim, M, codes[0], mags[0], F.astype(np.int8), codes[1], mags[1], 8, [A, B])
    assert (status == 0).all() and val[0] == -1.0 and -1.0 < val[1] <= 1.0
    # inside the search: every query filtered by F; nodes carrying B come back, nodes carrying A never do
    rng = np.random.default_rng(5)
    q = (vecs[rng.integers(0, 400, 32)] + 0.05 * rng.normal(size=(32, dim))).astype(np.float32).clip(-0.999, 0.999)
    filters = [[F.astype(np.int8)] for _ in range(32)]
    ix = md_index(vecs, mg, st, MK.Cosine)
    got, want = assert_filtered_equal(ix, mg, vecs, q, filters, k, ef)
    md_of = dict(zip(mg.node_id[0].tolist(), mg.node_md[0].tolist()))
    returned = [md_of[int(i)] for r in range(32) for i in want[0][r][: want[2][r]]]
    assert returned.count(3) > 0 and returned.count(2) == 0, (returned.count(3), returned.count(2))
    assert (mg.node_md[0] == 2).sum() > 0                     # A nodes exist and are dropped
    ix.close()


# ----------------------------------------------------------------------------- 6. filter rows per query
@gpu
def test_filter_rows_per_query_up_to_4096_and_the_refusal_past_it():
    st, dim, M, k, ef = ST.HalfPrecisionFP, 16, 16, 10, 128
    vecs, mg = mdgraph.build(n=400, dim=dim, md_dims=M, levels=3, nb=8, nb0=16, storage_type=int(st), metric=int(MK.Cosine),
                             seed=31, patterns=mdgraph.schema_patterns)
    rng = np.random.default_rng(8)
    q = (vecs[rng.integers(0, 400, 7)] + 0.05 * rng.normal(size=(7, dim))).astype(np.float32).clip(-0.999, 0.999)

    def rows(c):   # node patterns (strong matches exist) and random 0/1 rows
        return [mg.md_bits[2 + int(rng.integers(0, mg.md_bits.shape[0] - 2))].astype(np.int8) if rng.random() < 0.6
                else rng.integers(0, 2, M).astype(np.int8) for _ in range(c)]
    filters = [rows(1), rows(2), rows(33), rows(100), rows(4096), None, rows(3)]
    ix = md_index(vecs, mg, st, MK.Cosine)
    got, want = assert_filtered_equal(ix, mg, vecs, q, filters, k, ef)
    # (after the first filter row's traversal the kept fixed set stops the others at their entry, so a query whose first
    # row matches nothing may end empty, as in the reference)
    assert (want[3] == 0).all() and (want[2] > 0).sum() >= 3
    assert_same(device_search(ix, q, filters, k, ef), got)
    # 4097 rows: the host form refuses the call, the device form fails that query alone
    bad = list(filters)
    bad[4] = rows(4097)
    with pytest.raises(cdb.CosdataError) as e:
        ix.batch_search_filtered(q, bad, k, ef_search=ef, shortlist_size=64)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    ids, scores, counts, err = device_search(ix, q, bad, k, ef)
    assert err[4] == BAD_FILTER and counts[4] == 0
    keep = [0, 1, 2, 3, 5, 6]
    assert_same((ids[keep], scores[keep], counts[keep], err[keep]), tuple(a[keep] for a in got))
    ix.close()


# ----------------------------------------------------------------------------- 7 (GPU). the carve at 200 KB
@gpu
def test_metadata_carve_accepts_and_refuses_one_step_apart():
    ok, bad = carve_edge()
    st, k, ef = ST.FullPrecisionFP, 5, CARVE_EF
    for M in (ok, bad):
        vecs, mg = mdgraph.build(n=150, dim=CARVE_D, md_dims=M, levels=2, nb=8, nb0=16, storage_type=int(st),
                                 metric=int(MK.Cosine), seed=3, patterns=mdgraph.schema_patterns)
        q, filters = mdgraph.make_queries(vecs, mg, 8, seed=4)
        ix = md_index(vecs, mg, st, MK.Cosine)
        if M == ok:
            got, want = assert_filtered_equal(ix, mg, vecs, q, filters, k, ef)
            assert (want[2] > 0).sum() >= 2
        else:
            before = cdb.kernel_launch_count()
            with pytest.raises(cdb.CosdataError) as e:
                ix.batch_search_filtered(q, filters, k, ef_search=ef, shortlist_size=64)
            assert e.value.status == cdb.Status.INVALID_PARAMS and "shared memory" in str(e.value)
            assert cdb.kernel_launch_count() == before                   # refused before any kernel ran
            got, want = assert_filtered_equal(ix, mg, vecs, q, filters, k, 64)   # the same index at ef 64
        ix.close()


# ----------------------------------------------------------------------------- 8. replica writers at width
@gpu
@pytest.mark.parametrize("M", [33, 257])
def test_replica_build_insert_delete_at_metadata_width(M):
    from tests.test_gpu_hnsw_delete_replicas import assert_equal_to_oracle
    st, metric, dim, levels, nb, nb0, efc = ST.HalfPrecisionFP, MK.Cosine, 16, 3, 8, 16, 64
    n, n_a = 260, 170
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=M, levels=levels, seed=M, patterns=mdgraph.schema_patterns)
    cols = ("row", "node_id", "base_id", "md_row", "max_level")
    in_b = (pop["row"] != EMPTY) & (pop["row"] >= n_a)
    a = {c: pop[c][~in_b] for c in cols}
    b = {c: pop[c][in_b].copy() for c in cols}
    b["row"] += 2                                                        # behind the two roots the build appends
    vecs = pop["vecs"]
    ix = cdb.DenseIndex(dim=dim, storage_type=st, metric=metric, capacity=n + 2, keep_raw_f32=True)
    ix.append(vecs[:n_a])
    fa = ix.build_graph_replicas(a["row"], a["node_id"], a["base_id"], a["md_row"], a["max_level"], pop["md_bits"], pop["md_mags"],
                                 pop["main_root_md"], pop["pseudo_root_md"], levels, nb, nb0, efc, 64, 1, 1)
    ix.append(vecs[n_a:])
    codes, mags = ix.read_codes(0, n + 2)
    og = pydelete_md.Graph(metric, st, dim, codes, mags, pop["md_bits"], pop["md_mags"], levels, nb, nb0, n_a, pop["main_root_md"],
                           n_a + 1, pop["pseudo_root_md"])
    assert np.array_equal(fa, og.insert(a["row"], a["node_id"], a["base_id"], a["md_row"], a["max_level"], efc))
    assert_equal_to_oracle(ix, og, levels, int(metric), set(a["node_id"][fa != 0].tolist()))
    fb = ix.insert_graph_replicas(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], ef_construction=efc,
                                  shortlist_size=64, max_batch=1)
    assert np.array_equal(fb, og.insert(b["row"], b["node_id"], b["base_id"], b["md_row"], b["max_level"], efc))
    drop = set(a["node_id"][fa != 0].tolist()) | set(b["node_id"][fb != 0].tolist())
    assert_equal_to_oracle(ix, og, levels, int(metric), drop)
    rng = np.random.default_rng(M)
    rows = [int(r) for r in rng.choice(np.r_[0:n_a, n_a + 2:n + 2], 30, replace=False)]
    rows.append(rows[0])                                                 # deleted twice: status 1
    s = ix.delete_rows_replicas(rows, max_batch=1)
    assert np.array_equal(s, og.delete(rows)) and s[-1] == 1
    assert_equal_to_oracle(ix, og, levels, int(metric), drop)
    # with schema patterns the metadata replicas really are wide: some differ from each other beyond dim 32
    wide = pop["md_bits"][2:, 32:]
    assert (wide != wide[:1]).any()
    ix.close()
    og.close()
