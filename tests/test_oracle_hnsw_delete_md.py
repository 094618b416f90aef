"""The replica delete oracle (tests/hnsw_delete_md_oracle.c) against a pure-Python restatement of delete_embedding on a graph
with metadata (vector_store.rs:1206-1371 with the replica arms of cosine.rs:34-102 and the edge rules of :1014-1040) and
the deviations D1-D5 of cdb_index_delete_rows_replicas; and the oracle's continued insert against the pinned replica build."""
import heapq

import numpy as np
import pytest

import oracle as orc
from oracle import pymeta
from tests import mdgraph, pydelete_md

ST_F16, ST_U8, ST_SUB2 = 4, 0, 2
COS, DOT = 0, 3
EMPTY = 0xFFFFFFFF
OK = 0


def population(st, metric, n=160, dim=16, levels=3, seed=3, zero=None):
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=seed)
    vecs = pop["vecs"].copy()
    if zero is not None:
        vecs[zero] = 0.0
    root = np.linspace(-0.9, 0.9, dim).astype(np.float32)
    codes, mags = orc.quantize_batch(st, np.concatenate([vecs, root[None], np.zeros((1, dim), np.float32)]))
    row = np.where(pop["row"] == EMPTY, n + 1, pop["row"]).astype(np.uint32)
    return pop, codes, mags, row


def oracle_graph(st, metric, pop, codes, mags, levels, nb, nb0):
    n = pop["vecs"].shape[0]
    return pydelete_md.Graph(metric, st, pop["vecs"].shape[1], codes, mags, pop["md_bits"], pop["md_mags"], levels, nb, nb0, n,
                             pop["main_root_md"], n + 1, pop["pseudo_root_md"])


@pytest.mark.parametrize("st,metric", [(ST_F16, COS), (ST_SUB2, DOT)])
def test_continued_insert_equals_the_replica_build(st, metric):
    levels, nb, nb0, efc = 3, 4, 8, 24
    pop, codes, mags, row = population(st, metric, zero=8)
    n = pop["vecs"].shape[0]
    rl = pymeta.ReplicaList(row, pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], n, pop["main_root_md"], n + 1,
                            pop["pseudo_root_md"])
    mg, failed = pymeta.build_md(metric, st, pop["vecs"].shape[1], codes, mags, pop["md_bits"], pop["md_mags"], rl, num_levels=levels,
                                 neighbors_count=nb, level0_neighbors_count=nb0, ef_construction=efc)
    g = oracle_graph(st, metric, pop, codes, mags, levels, nb, nb0)
    cuts = [0, 40, 41, row.size // 2, row.size]
    got = np.concatenate([g.insert(pop["row"][a:b], pop["node_id"][a:b], pop["base_id"][a:b], pop["md_row"][a:b], pop["max_level"][a:b],
                                   efc) for a, b in zip(cuts, cuts[1:])])
    assert np.array_equal(got, failed) and (metric != COS or failed.any())
    e = g.export()
    for lv in range(levels + 1):
        assert np.array_equal(e["node_row"][lv], mg.fg.node_row[lv]), lv
        assert np.array_equal(e["adj"][lv], mg.fg.adj[lv]), lv
        assert np.array_equal(e["node_id"][lv], mg.node_id[lv]) and np.array_equal(e["node_md"][lv], mg.node_md[lv]), lv
        if lv:
            assert np.array_equal(e["child"][lv], mg.fg.child[lv]), lv
        ids = dict(zip(pop["node_id"].tolist(), range(row.size)))
        assert all(e["ins"][lv][j] == ids[int(e["node_id"][lv][j])] for j in range(2, e["ins"][lv].size)), lv
    g.close()


class PyMd:
    """the exported replica graph with the reference's node operations, in plain Python"""

    def __init__(self, e, g, entries):
        self.g, self.entries = g, entries
        self.L1 = g.num_levels + 1
        self.nb = [g.nbrs0] + [g.nbrs] * g.num_levels
        self.min_key = orc.order_key(g.metric, -1.0 if g.metric == COS else -np.inf)
        self.max_key = orc.order_key(g.metric, 2.0 if g.metric == COS else np.inf)
        self.node_row = [list(map(int, a)) for a in e["node_row"]]
        self.node_id = [list(map(int, a)) for a in e["node_id"]]
        self.node_md = [list(map(int, a)) for a in e["node_md"]]
        self.ins = [list(map(int, a)) for a in e["ins"]]
        self.child = [list(map(int, a)) for a in e["child"]]
        self.adj = [[list(map(int, a[i * nb:(i + 1) * nb])) for i in range(len(a) // nb)] for a, nb in zip(e["adj"], self.nb)]
        self.sk = [[list(map(int, a[i * nb:(i + 1) * nb])) for i in range(len(a) // nb)] for a, nb in zip(e["simkey"], self.nb)]
        self.li = [list(map(int, a)) for a in e["lowest_idx"]]
        self.lk = [list(map(int, a)) for a in e["lowest_key"]]
        self.relinks, self.rule_skips, self.unreachable = 0, 0, 0
        self.skips_add_neighbor_refuses = 0   # rule skips that ProbNode::add_neighbor would have refused anyway

    def vd(self, row, vid, md):
        g = self.g
        return pymeta.VectorData(g.codes[row], g.mags[row], vid, None if md == EMPTY else g.md_bits[md],
                                 0.0 if md == EMPTY else g.md_mags[md])

    def side(self, L, node):
        return self.vd(self.node_row[L][node], self.node_id[L][node], self.node_md[L][node])

    def calc(self, x, y):
        return pymeta.distance_md(self.g.metric, self.g.st, self.g.dim, self.g.md_bits.shape[1], x, y)

    def key(self, score, ident):
        return (orc.order_key(self.g.metric, float(score)) << 32) | (~ident & 0xFFFFFFFF)

    def kind(self, L, node):
        return pymeta.replica_kind(self.side(L, node))

    def traverse(self, L, entry, x, shortlist):
        """traverse_find_nearest, a fresh fixed set with nothing pre-inserted, ef 512, best 100 -> (rc, [(key, node, score)])"""
        nb = self.nb[L]
        fs = [0] * nb
        member = lambda v: (fs[(v >> 6) & (nb - 1)] >> (v & 63)) & 1

        def insert(v):
            fs[(v >> 6) & (nb - 1)] |= 1 << (v & 63)
        rc, d = self.calc(x, self.side(L, entry))
        if rc != OK:
            return rc, []
        insert(self.node_id[L][entry])
        heap, res, visited = [(-self.key(d, self.node_id[L][entry]), entry, d)], [], 0
        while heap:
            k, node, d = heapq.heappop(heap)
            if visited >= 512:
                break
            visited += 1
            res.append((-k, node, d))
            for s in range(min(shortlist, nb)):
                nbl = self.adj[L][node][s]
                if nbl == EMPTY or member(self.node_id[L][nbl]):
                    continue
                rc, d = self.calc(x, self.side(L, nbl))
                if rc != OK:
                    return rc, []
                insert(self.node_id[L][nbl])
                heapq.heappush(heap, (-self.key(d, self.node_id[L][nbl]), nbl, d))
        res.sort(reverse=True)
        return OK, res[:100]

    def add_neighbor(self, L, node, nbr, dkey):
        adj, sk = self.adj[L][node], self.sk[L][node]
        lidx, lkey = self.li[L][node], self.lk[L][node]
        if dkey <= lkey:
            return None
        ok, old = False, EMPTY
        if adj[lidx] == EMPTY:
            adj[lidx], sk[lidx], ok = nbr, dkey, True
        elif dkey > sk[lidx]:
            old, adj[lidx], sk[lidx], ok = adj[lidx], nbr, dkey, True
        nidx, nkey = 0, self.max_key
        for s in range(self.nb[L]):
            if adj[s] == EMPTY:
                nidx, nkey = s, self.min_key
                break
            if sk[s] < nkey:
                nidx, nkey = s, sk[s]
        self.li[L][node], self.lk[L][node] = nidx, nkey
        if not ok:
            return None
        if old != EMPTY:
            self.remove_by_id(L, old, node)
        return lidx

    def remove_by_id(self, L, node, ident):
        a = self.adj[L][node]
        for s in range(self.nb[L]):
            if a[s] == ident:
                a[s] = EMPTY
                return True
        return False

    def create_node_edges(self, L, node, cands):
        """with the replica rules (cosine): a Metadata node takes a Pseudo neighbour only at 1.0, never a Metadata one at -1.0"""
        nk, successful = self.kind(L, node), 0
        for key, nbr, score in cands:
            if successful >= self.nb[L]:
                break
            if self.g.metric == COS and nk == pymeta.KIND_METADATA:
                bk = self.kind(L, nbr)
                if (bk == pymeta.KIND_PSEUDO and score != 1.0) or (bk == pymeta.KIND_METADATA and score == -1.0):
                    self.rule_skips += 1
                    self.skips_add_neighbor_refuses += (key >> 32) <= self.lk[L][node]
                    continue
            idx = self.add_neighbor(L, node, nbr, key >> 32)
            if idx is None:
                continue
            if self.add_neighbor(L, nbr, node, key >> 32) is not None:
                successful += 1
            elif self.adj[L][node][idx] == nbr:
                self.adj[L][node][idx] = EMPTY

    def dead(self, L, node, r):
        return node >= 2 and self.node_row[L][node] == r

    def relink(self, L, N, D, results, r):
        x, cands = self.side(L, N), []
        for _, c, _ in results:
            if c in (D, N) or self.dead(L, c, r):
                continue
            rc, d = self.calc(x, self.side(L, c))
            if rc != OK:
                self.unreachable += rc == pymeta.UNREACHABLE
                return rc
            cands.append((self.key(d, self.node_id[L][c]), c, d))
        cands.sort(reverse=True)
        self.relinks += 1
        self.create_node_edges(L, N, cands)
        return OK

    def delete(self, r, deleted, shortlist):
        if deleted[r]:
            return 1
        deleted[r] = 1
        items = [t for t, e in enumerate(self.entries) if e[0] == r]
        if not items:
            return 0
        status, res, loc = 0, {}, {}
        for k, t in enumerate(items):   # every node traverses the graph as of the row's start
            _, vid, md = self.entries[t]
            x = self.vd(r, vid, md)
            entry = 1 if md != EMPTY and self.g.md_mags[md] != 0 else 0
            err = False
            for L in range(self.L1 - 1, -1, -1):
                loc[k, L] = next((j for j in range(2, len(self.ins[L])) if self.ins[L][j] == t), None)
                if err:
                    res[k, L] = None
                    continue
                rc, rs = self.traverse(L, entry, x, shortlist)
                if rc != OK:
                    err, status, res[k, L] = True, 2, None
                    continue
                res[k, L] = rs
                if L > 0:
                    entry = self.child[L][rs[0][1]]
        for L in range(self.L1):
            for k in range(len(items)):   # list order
                D = loc[k, L]
                if D is None:
                    continue
                for s in range(self.nb[L]):
                    N = self.adj[L][D][s]
                    if N == EMPTY:
                        continue
                    if self.remove_by_id(L, N, D) and not self.dead(L, N, r) and all(a == EMPTY for a in self.adj[L][N]) \
                            and res[k, L] is not None and self.relink(L, N, D, res[k, L], r) != OK:
                        status = 2
                self.adj[L][D] = [EMPTY] * self.nb[L]
                self.li[L][D], self.lk[L][D] = 0, self.min_key
            first = {}
            for x, a in enumerate(self.adj[L]):   # D2
                for s in range(self.nb[L]):
                    if a[s] != EMPTY and self.dead(L, a[s], r):
                        k = next(k for k in range(len(items)) if loc[k, L] == a[s])
                        first[x] = min(first.get(x, k), k)
                        a[s] = EMPTY
            for x in sorted(first):
                k = first[x]
                if not self.dead(L, x, r) and all(a == EMPTY for a in self.adj[L][x]) and res[k, L] is not None and \
                        self.relink(L, x, loc[k, L], res[k, L], r) != OK:
                    status = 2
        return status


def build(st, metric, levels=3, nb=4, nb0=8, efc=24, zero=None, n=160):
    pop, codes, mags, row = population(st, metric, n=n, zero=zero)
    g = oracle_graph(st, metric, pop, codes, mags, levels, nb, nb0)
    failed = g.insert(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], efc)
    entries = list(zip(row.tolist(), pop["node_id"].tolist(), pop["md_row"].tolist()))
    return g, pop, entries, failed


def run_both(g, entries, rows, shortlist=64):
    p = PyMd(g.export(), g, entries)
    pdel = g.deleted.copy()
    want = np.array([p.delete(int(r), pdel, shortlist) for r in rows], np.uint8)
    got = g.delete(rows, shortlist)
    assert np.array_equal(got, want)
    assert np.array_equal(g.deleted, pdel)
    e = g.export()
    for L in range(g.num_levels + 1):
        adj = np.array([x for a in p.adj[L] for x in a], np.uint32)
        assert np.array_equal(e["adj"][L], adj), L
        sk = np.array([x for a in p.sk[L] for x in a], np.uint32)
        assert np.array_equal(e["simkey"][L][adj != EMPTY], sk[adj != EMPTY]), L
        assert np.array_equal(e["lowest_idx"][L], np.array(p.li[L], np.uint32)), L
        assert np.array_equal(e["lowest_key"][L], np.array(p.lk[L], np.uint32)), L
    return p, got


def no_links_to(g, rows):
    e = g.export()
    dead = set(int(r) for r in rows)
    for L in range(g.num_levels + 1):
        nb = g.nbrs0 if L == 0 else g.nbrs
        adj = e["adj"][L].reshape(-1, nb)
        nr = e["node_row"][L]
        for i in range(2, adj.shape[0]):
            assert not dead.intersection(int(nr[a]) for a in adj[i] if a != EMPTY), (L, i)
            if int(nr[i]) in dead:
                assert (adj[i] == EMPTY).all(), (L, i)


def pick_rows(pop, n, rng, count):
    """rows with only a base replica, with one and with two Metadata replicas, mixed"""
    reps = np.bincount(pop["row"][pop["row"] != EMPTY], minlength=n)
    groups = [np.flatnonzero(reps == c) for c in (1, 2, 3)]
    assert all(gr.size for gr in groups)
    return np.concatenate([rng.choice(gr, count // 3, replace=False) for gr in groups])


@pytest.mark.parametrize("st,metric", [(ST_F16, COS), (ST_U8, COS), (ST_SUB2, DOT)])
def test_oracle_equals_restatement(st, metric):
    g, pop, entries, failed = build(st, metric, nb=2, nb0=2)   # small lists: neighbours empty and are relinked
    n = pop["vecs"].shape[0]
    rows = pick_rows(pop, n, np.random.default_rng(1), 45)
    rows = np.random.default_rng(2).permutation(rows)
    p, status = run_both(g, entries, rows)
    assert p.relinks > 5
    no_links_to(g, rows)
    # the second call: duplicates, rows deleted before, fresh rows
    more = [int(rows[0]), int(rows[0])] + [int(r) for r in pick_rows(pop, n, np.random.default_rng(3), 9) if r not in rows][:5]
    p, status = run_both(g, entries, more)
    assert status[0] == 1 and status[1] == 1
    no_links_to(g, list(rows) + more)
    g.close()


def twin_population(n=400, dim=32, levels=2, seed=23):
    """replica_population with weighted dimensions: every pattern is scaled by 10, and an embedding with two Metadata
    replicas gets its second one on a twin of its first pattern (the same dims plus 1 on a dimension the pattern leaves at
    0: cosine 0.995 > 0.99).  The two replicas of such a row then score each other and share neighbours, so the order in
    which a delete repairs them matters."""
    pop = mdgraph.replica_population(n=n, dim=dim, md_dims=6, levels=levels, seed=seed)
    base = pop["md_bits"][2:] * 10
    twins = base.copy()
    twins[:, 5] += 1
    assert (base[:, 5] == 0).all()
    bits_ = np.concatenate([pop["md_bits"][:2], base, twins]).astype(np.int32)
    mags_ = np.array([pymeta.metadata_mag(r) for r in bits_], np.float32)
    mags_[0] = 0.0
    md = pop["md_row"].copy()
    n_pat = base.shape[0]
    for r in np.unique(pop["row"][pop["row"] != EMPTY]):
        t = np.flatnonzero((pop["row"] == r) & (pop["md_row"] >= 2))
        if t.size == 2:
            md[t[1]] = md[t[0]] + n_pat
    return dict(pop, md_bits=bits_, md_mags=mags_, md_row=md)


def early_and_more_metadata_rows(pop, n, more, seed=7):
    """the first 24 embeddings with Metadata replicas (their replicas fill the pseudo nodes' slots at cs == 1.0, so deleting
    them empties pseudo nodes), then `more` other embeddings with Metadata replicas"""
    reps = np.bincount(pop["row"][pop["row"] != EMPTY], minlength=n)
    md_rows = np.flatnonzero(reps > 1)
    return [int(r) for r in md_rows[:24]] + [int(r) for r in np.random.default_rng(seed).permutation(md_rows[24:])[:more]]


@pytest.mark.parametrize("st", [ST_F16, ST_U8])
def test_replica_relinks_rules_and_unreachable_arm(st):
    """parameters where D5's relink paths all run: Metadata and Pseudo nodes empty and are relinked, the edge rules skip
    candidates, and a Pseudo node rescoring a Metadata candidate hits the unreachable arm (status 2 without any zero-norm row)"""
    n, dim = 400, 32
    pop = twin_population(n, dim)
    root = np.linspace(-0.9, 0.9, dim).astype(np.float32)
    codes, mags = orc.quantize_batch(st, np.concatenate([pop["vecs"], root[None], np.zeros((1, dim), np.float32)]))
    row = np.where(pop["row"] == EMPTY, n + 1, pop["row"]).astype(np.uint32)
    g = oracle_graph(st, COS, pop, codes, mags, 2, 4, 8)
    assert not g.insert(pop["row"], pop["node_id"], pop["base_id"], pop["md_row"], pop["max_level"], 32).any()
    entries = list(zip(row.tolist(), pop["node_id"].tolist(), pop["md_row"].tolist()))
    rows = early_and_more_metadata_rows(pop, n, 230)
    p, status = run_both(g, entries, rows)
    assert p.relinks > 20 and p.rule_skips > 0 and p.unreachable > 0
    assert (status == 2).sum() == p.unreachable                         # every status 2 is a relink Err
    # every candidate the rules skip scores MetricResult::min (-1), which add_neighbor refuses as well: the rules never
    # change a relink's outcome here, they only keep it from being attempted (as in the reference)
    assert p.skips_add_neighbor_refuses == p.rule_skips
    no_links_to(g, rows)
    g.close()


def test_zero_norm_row():
    pop0 = mdgraph.replica_population(n=160, dim=16, md_dims=6, levels=3, seed=3)
    reps = np.bincount(pop0["row"][pop0["row"] != EMPTY], minlength=160)
    zero = int(np.flatnonzero(reps == 3)[0])
    g, pop, entries, failed = build(ST_F16, COS, nb=2, nb0=2, zero=zero)
    assert failed.any()                                                  # its base replica's insert failed
    rows = [zero] + [int(r) for r in pick_rows(pop, 160, np.random.default_rng(5), 45) if r != zero]
    p, status = run_both(g, entries, rows)
    assert status[0] == 2
    no_links_to(g, rows)
    g.close()


def test_python_argument_checks():
    """DenseIndex.delete_rows_replicas checks its arguments on the host, before the library is called"""
    import types
    import cosdata_b200 as cdb
    fake = types.SimpleNamespace(size=10)
    for rows, kw in (([[1, 2]], {}), ([-1], {}), ([10], {}), ([1], dict(shortlist_size=0)), ([1], dict(shortlist_size=65))):
        with pytest.raises(ValueError):
            cdb.DenseIndex.delete_rows_replicas(fake, rows, **kw)
