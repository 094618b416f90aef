"""The delete oracle (tests/hnsw_delete_oracle.c) against a pure-Python restatement of delete_embedding
(src/vector_store.rs:1206-1371, ProbNode::add_neighbor / remove_neighbor_by_id, create_node_edges) with the deviations
D1-D4 of cdb_index_delete_rows, on small graphs built by the insert oracle or uploaded by hand."""
import ctypes as C
import heapq

import numpy as np
import pytest

import oracle as orc
from tests import pydelete, pyinsert

ST_F16, ST_U8, ST_SUB2 = 4, 0, 2
COS, DOT = 0, 3
EMPTY = 0xFFFFFFFF
ROOT_ID = 0xFFFFFFFF
OK = 0


class PyGraph:
    """the exported graph (dict of Graph.export) with the reference's node operations, in plain Python"""

    def __init__(self, e, metric, st, dim, codes, mags):
        self.metric, self.st, self.dim, self.codes, self.mags = metric, st, dim, codes, mags
        self.root_row, self.entry, self.num_levels = e["root_row"], e["entry"], e["num_levels"]
        self.min_key, self.max_key = pyinsert.min_max_keys(metric)
        self.nb = [e["level0_neighbors_count"]] + [e["neighbors_count"]] * self.num_levels
        self.node_row = [list(map(int, a)) for a in e["node_row"]]
        self.child = [list(map(int, a)) for a in e["child"]]
        self.adj = [[list(map(int, a[i * nb:(i + 1) * nb])) for i in range(len(a) // nb)] for a, nb in zip(e["adj"], self.nb)]
        self.sk = [[list(map(int, a[i * nb:(i + 1) * nb])) for i in range(len(a) // nb)] for a, nb in zip(e["simkey"], self.nb)]
        self.li = [list(map(int, a)) for a in e["lowest_idx"]]
        self.lk = [list(map(int, a)) for a in e["lowest_key"]]
        self.found, self.missed, self.relinks, self.stale_refusals, self.swept = 0, 0, 0, 0, 0

    def ident(self, row):
        return ROOT_ID if row == self.root_row else row

    def _calc(self, x, y):
        """DistanceMetric::calculate on two stored rows -> (rc, score)"""
        out = np.zeros(1, np.float32)
        rc = orc.pyoracle.lib().orc_distance(self.metric, self.st, self.dim, self.codes[x].ctypes.data_as(C.c_void_p),
                                             float(self.mags[x]), self.codes[y].ctypes.data_as(C.c_void_p), float(self.mags[y]),
                                             out.ctypes.data_as(C.POINTER(C.c_float)))
        return rc, float(out[0])

    def key(self, score, ident):
        return (orc.order_key(self.metric, score) << 32) | (~ident & 0xFFFFFFFF)

    def traverse(self, L, entry, q, ef, shortlist, final_len):
        """traverse_find_nearest with a fresh PerformantFixedSet and nothing pre-inserted -> (rc, [(key, node)])"""
        nb = self.nb[L]
        fs = [0] * nb

        def member(v):
            return (fs[(v >> 6) & (nb - 1)] >> (v & 63)) & 1

        def insert(v):
            fs[(v >> 6) & (nb - 1)] |= 1 << (v & 63)

        erow = self.node_row[L][entry]
        rc, d = self._calc(q, erow)
        if rc != OK:
            return rc, []
        insert(self.ident(erow))
        heap, res, visited = [(-self.key(d, self.ident(erow)), entry)], [], 0
        while heap:
            k, node = heapq.heappop(heap)
            if visited >= ef:
                break
            visited += 1
            res.append((-k, node))
            for s in range(min(shortlist, nb)):
                nbl = self.adj[L][node][s]
                if nbl == EMPTY:
                    continue
                nrow = self.node_row[L][nbl]
                if member(self.ident(nrow)):
                    continue
                rc, d = self._calc(q, nrow)
                if rc != OK:
                    return rc, []
                insert(self.ident(nrow))
                heapq.heappush(heap, (-self.key(d, self.ident(nrow)), nbl))
        res.sort(reverse=True)
        return OK, res[:final_len]

    def add_neighbor(self, L, node, nbr, dkey, count_stale=False):
        """ProbNode::add_neighbor (prob_node.rs:210-283) -> slot or None"""
        adj, sk = self.adj[L][node], self.sk[L][node]
        lidx, lkey = self.li[L][node], self.lk[L][node]
        if dkey <= lkey:
            if count_stale and all(a == EMPTY for a in adj) and lkey != self.min_key:
                self.stale_refusals += 1
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
        successful = 0
        for key, nbr in cands:
            if successful >= self.nb[L]:
                break
            dkey = key >> 32
            idx = self.add_neighbor(L, node, nbr, dkey, count_stale=True)
            if idx is None:
                continue
            if self.add_neighbor(L, nbr, node, dkey) is not None:
                successful += 1
            elif self.adj[L][node][idx] == nbr:
                self.adj[L][node][idx] = EMPTY

    def relink(self, L, N, D, results, deleted):
        nrow = self.node_row[L][N]
        cands = []
        for _, c in results:
            crow = self.node_row[L][c]
            if c in (D, N) or deleted[crow]:
                continue
            rc, d = self._calc(nrow, crow)
            if rc != OK:
                return rc
            cands.append((self.key(d, self.ident(crow)), c))
        cands.sort(reverse=True)
        self.relinks += 1
        self.create_node_edges(L, N, cands)
        return OK

    def delete(self, r, deleted, shortlist):
        """delete_embedding for row r -> status (0 deleted, 1 already deleted, 2 an Err stopped relinks)"""
        if deleted[r]:
            return 1
        deleted[r] = 1
        if r >= len(self.node_row[0]):
            return 0
        status, err, entry = 0, False, self.entry
        for L in range(self.num_levels, -1, -1):
            results = []
            if not err:
                rc, results = self.traverse(L, entry, r, 512, shortlist, 100)   # ef 512, final_len 100
                if rc != OK:
                    err, status = True, 2
                elif L > 0:
                    entry = self.child[L][results[0][1]]
            rows = self.node_row[L]
            D = r if L == 0 else next((j for j, x in enumerate(rows) if x == r), None)
            if D is None:
                continue
            if not err:
                if any(n == D for _, n in results):
                    self.found += 1
                else:
                    self.missed += 1
            for s in range(self.nb[L]):   # D's own slots, read as the loop reaches them
                N = self.adj[L][D][s]
                if N == EMPTY:
                    continue
                if self.remove_by_id(L, N, D) and not deleted[rows[N]] and all(a == EMPTY for a in self.adj[L][N]) and not err:
                    if self.relink(L, N, D, results, deleted) != OK:
                        status = 2
            self.adj[L][D] = [EMPTY] * self.nb[L]
            self.li[L][D], self.lk[L][D] = 0, self.min_key
            touched = []
            for x, a in enumerate(self.adj[L]):   # D2
                hit = [s for s in range(self.nb[L]) if a[s] == D]
                for s in hit:
                    a[s] = EMPTY
                if hit:
                    touched.append(x)
            self.swept += len(touched)
            for x in touched:
                if not deleted[rows[x]] and all(a == EMPTY for a in self.adj[L][x]) and not err:
                    if self.relink(L, x, D, results, deleted) != OK:
                        status = 2
        return status


def clustered(n, dim, seed):
    rng = np.random.default_rng(seed)
    centres = rng.normal(size=(8, dim)).astype(np.float32)
    v = (centres[rng.integers(0, 8, n)] + 0.35 * rng.normal(size=(n, dim))).astype(np.float32)
    return (v / (np.abs(v).max() * 1.01)).astype(np.float32)


def built(metric, st, n, dim, levels, nb, nb0, seed, zero_rows=()):
    vecs = clustered(n, dim, seed)
    for z in zero_rows:
        vecs[z] = 0.0
    root = np.linspace(-0.9, 0.9, dim).astype(np.float32)
    codes, mags = orc.quantize_batch(st, np.concatenate([vecs, root[None]]).astype(np.float32))
    g = pydelete.Graph.init(metric, st, dim, codes, mags, n, levels, nb, nb0)
    g.insert(0, n, ef_construction=24, seed=seed)
    return g, codes, mags


def assert_same(g, p):
    e = g.export()
    for L in range(g.num_levels + 1):
        nb = p.nb[L]
        adj = np.array([x for a in p.adj[L] for x in a], np.uint32)
        assert np.array_equal(e["adj"][L], adj), L
        filled = adj != EMPTY
        sk = np.array([x for a in p.sk[L] for x in a], np.uint32)
        assert np.array_equal(e["simkey"][L][filled], sk[filled]), L
        assert np.array_equal(e["lowest_idx"][L], np.array(p.li[L], np.uint32)), L
        assert np.array_equal(e["lowest_key"][L], np.array(p.lk[L], np.uint32)), L
        assert nb == (g.nbrs0 if L == 0 else g.nbrs)


def run_both(g, codes, mags, rows, shortlist=64):
    p = PyGraph(g.export(), g.metric, g.st, g.dim, codes, mags)
    pdel = g.deleted.copy()
    want = np.array([p.delete(int(r), pdel, shortlist) for r in rows], np.uint8)
    got = g.delete(rows, shortlist)
    assert np.array_equal(got, want)
    assert np.array_equal(g.deleted, pdel)
    assert_same(g, p)
    return p, got


def no_links_to(g, rows):
    e = g.export()
    dead = set(int(r) for r in rows)
    for L in range(g.num_levels + 1):
        nb = g.nbrs0 if L == 0 else g.nbrs
        adj = e["adj"][L].reshape(-1, nb)
        nr = e["node_row"][L]
        for i in range(adj.shape[0]):
            named = [int(nr[a]) for a in adj[i] if a != EMPTY]
            assert not dead.intersection(named), (L, i)
            if int(nr[i]) in dead:
                assert (adj[i] == EMPTY).all(), (L, i)


@pytest.mark.parametrize("st,metric", [(ST_F16, COS), (ST_U8, COS), (ST_SUB2, DOT), (ST_F16, DOT)])
def test_oracle_equals_restatement(st, metric):
    n, dim = 300, 16
    g, codes, mags = built(metric, st, n, dim, 3, 4, 8, 5)
    rows = np.random.default_rng(1).choice(n, 32, replace=False)
    p, status = run_both(g, codes, mags, rows)
    assert (status == 0).all()
    assert p.found > 0 and p.relinks > 0
    no_links_to(g, rows)
    g.close()


def test_missed_node_and_asymmetric_in_link():
    """an uploaded level-0 graph where D is reachable only through a one-way link from a node D does not list (D2), and a
    node that links D is never reached from the root (D1: D is missed there but still unlinked)"""
    n, dim, nb0 = 40, 16, 4
    vecs = clustered(n, dim, 3)
    root = np.linspace(-0.9, 0.9, dim).astype(np.float32)
    codes, mags = orc.quantize_batch(ST_F16, np.concatenate([vecs, root[None]]).astype(np.float32))
    adj = np.full((n + 1, nb0), EMPTY, np.uint32)
    for i in range(n):   # a ring over rows 0..29, the root linked both ways to row 0; rows 30..39 link into the ring only
        if i < 30:
            adj[i, 0], adj[i, 1] = (i + 1) % 30, (i - 1) % 30
        else:
            adj[i, 0] = i - 30
    adj[n, 0], adj[0, 2] = 0, n
    e = dict(num_levels=0, neighbors_count=nb0, level0_neighbors_count=nb0, entry=n, root_row=n,
             node_row=[np.arange(n + 1, dtype=np.uint32)], adj=[adj.ravel()], child=[np.zeros(n + 1, np.uint32)])
    g = pydelete.Graph.from_graph(COS, ST_F16, dim, codes, mags, e)
    p, status = run_both(g, codes, mags, [5, 33, 12])
    assert (status == 0).all()
    assert p.missed >= 1 and p.swept >= 1
    no_links_to(g, [5, 33, 12])
    g.close()


def test_zero_norm_row_and_repeat_delete():
    n, dim = 200, 16
    g, codes, mags = built(COS, ST_F16, n, dim, 2, 4, 8, 9, zero_rows=(17,))
    p, status = run_both(g, codes, mags, [17, 3, 3, 17, 40])
    assert list(status) == [2, 0, 1, 1, 0]
    p, status = run_both(g, codes, mags, [3, 40])
    assert list(status) == [1, 1]
    g.close()


def test_delete_everything_but_the_root():
    n, dim = 120, 16
    g, codes, mags = built(DOT, ST_F16, n, dim, 2, 4, 8, 4)
    rows = np.random.default_rng(3).permutation(n)
    p, status = run_both(g, codes, mags, rows)
    assert (status == 0).all()
    assert p.stale_refusals > 0   # an emptied node refused a candidate no better than the similarity it lost
    e = g.export()
    for L in range(g.num_levels + 1):
        assert (e["adj"][L] == EMPTY).all(), L
    g.close()
