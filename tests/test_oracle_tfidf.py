"""The TF-IDF oracle (tests/tfidf_oracle.c) against a pure-Python restatement of the reference: VersionedVec with packed
u64 words (versioned_vec.rs), N, get_idf with the C library's log1pf, and search_bm25 with Rust std's BinaryHeap
(sparse_ann_query.rs:149-302).  Also: the oracle's `query` summation order against its `heap` order, the df wrap after
cross-version deletes, the BM25 term-frequency helpers, and the absence of a CPU fallback."""
import ctypes as C
import ctypes.util
from fractions import Fraction

import numpy as np
import pytest

import cosdata_b200 as cdb
from tests import pytfidf as pt
from tests.tfidf_data import op_script, query_csr, random_queries

MAX = (1 << 64) - 1
_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.log1pf.restype = C.c_float
_libm.log1pf.argtypes = [C.c_float]
f32 = np.float32


def get_idf(n, df):
    num = f32((n - df) % (1 << 32)) + f32(0.5)
    den = f32(df) + f32(0.5)
    return f32(_libm.log1pf(float(f32(num / den))))


def bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def from_bits(b):
    return np.array([b], np.uint32).view(np.float32)[0]


def total_key(x):
    b = bits(x)
    return (~b & 0xFFFFFFFF) if b & 0x80000000 else b | 0x80000000


class Unreachable(Exception):
    pass


class VersionedVec:
    """versioned_vec.rs: a chain of (version, [u64 word]) segments"""

    def __init__(self, version):
        self.segs = [[version, []]]

    def _seg(self, version):
        for s in self.segs:
            if s[0] == version:
                return s
        s = [version, []]
        self.segs.append(s)
        return s

    def push_sorted(self, version, doc, tf):
        lst = self._seg(version)[1]
        i = len(lst)
        while i > 0 and (lst[i - 1] >> 32) > doc:
            i -= 1
        lst.insert(i, (doc << 32) | bits(tf))

    def delete(self, version, doc):
        for s in self.segs:
            for idx, w in enumerate(s[1]):
                if (w >> 32) == doc:
                    s[1][idx] = MAX
                    ins = s[0]
                    t = self._seg(version)
                    if ins == version:
                        t[1].pop(idx)
                    else:
                        t[1].append((1 << 63) | (ins << 32) | idx)
                    return

    def __len__(self):
        return sum(len(s[1]) for s in self.segs)

    def iter(self):
        for s in self.segs:
            for w in s[1]:
                if w == MAX or w & (1 << 63):
                    continue
                yield (w >> 32, from_bits(w & 0xFFFFFFFF))


class Head:
    def __init__(self, vv, idf):
        self.it = vv.iter()
        self.nxt = next(self.it, None)
        self.idf = idf

    def peek(self):
        return self.nxt

    def pop(self):
        x = self.nxt
        if x is not None:
            self.nxt = next(self.it, None)
        return x


def le(a, b):
    """a <= b under PostingListHead's Ord (o.0.cmp(&s.0)), with its unreachable! on an exhausted head"""
    s, o = a.peek(), b.peek()
    if s is None or o is None:
        raise Unreachable
    return s[0] >= o[0]


def sift_up(d, start, pos):
    e = d[pos]
    while pos > start:
        parent = (pos - 1) // 2
        if le(e, d[parent]):
            break
        d[pos] = d[parent]
        pos = parent
    d[pos] = e


def heap_push(d, x):
    d.append(x)
    sift_up(d, 0, len(d) - 1)


def heap_pop(d):
    if not d:
        return None
    item = d.pop()
    if d:
        item, d[0] = d[0], item
        end, pos = len(d), 0
        e = d[0]
        child = 1
        while child <= max(end - 2, 0):
            child += 1 if le(d[child], d[child + 1]) else 0
            d[pos] = d[child]
            pos = child
            child = 2 * pos + 1
        if child == end - 1:
            d[pos] = d[child]
            pos = child
        d[pos] = e
        sift_up(d, 0, pos)
    return item


class PyIndex:
    """TFIDFIndex: insert / mark_embedding_as_deleted (a deleted row again is skipped, the documented deviation)"""

    def __init__(self, id_base=0):
        self.id_base, self.n, self.terms, self.rows = id_base, 0, {}, []

    def append(self, rows, counted, version):
        for r, pairs in enumerate(rows):
            doc = self.id_base + len(self.rows)
            self.rows.append([pairs, bool(counted[r]), False])
            if counted[r]:
                self.n += 1
            for h, tf in pairs:
                if h not in self.terms:
                    self.terms[h] = VersionedVec(version)
                self.terms[h].push_sorted(version, doc, f32(tf))

    def delete(self, rows, version):
        for r in rows:
            row = self.rows[int(r)]
            if row[2]:
                continue
            row[2] = True
            if not row[1]:
                continue
            self.n -= 1
            for h, _ in row[0]:
                self.terms[h].delete(version, self.id_base + int(r))

    def search_bm25(self, query, k):
        heads = []
        for h in query:
            if h in self.terms:
                vv = self.terms[h]
                heap_push(heads, Head(vv, get_idf(self.n, len(vv))))
        buckets = [(0xFFFFFFFF, f32(-np.inf))] * 512
        with np.errstate(all="ignore"):
            while heads:
                head = heap_pop(heads)
                x = head.pop()
                if x is None:
                    continue
                doc, tf = x
                score = f32(tf * head.idf)
                if head.peek() is not None:
                    heap_push(heads, head)
                while heads:
                    y = heads[0].peek()
                    if y is None:
                        heap_pop(heads)
                        continue
                    if y[0] != doc:
                        break
                    score = f32(score + f32(y[1] * heads[0].idf))
                    hh = heap_pop(heads)
                    hh.pop()
                    if hh.peek() is not None:
                        heap_push(heads, hh)
                b = doc % 512
                if score > buckets[b][1]:
                    buckets[b] = (doc, score)
        res = [x for x in buckets if x[0] != 0xFFFFFFFF]
        res.sort(key=lambda x: (-total_key(x[1]), x[0]))
        return res[:k] if k else res


def run_script(seed, id_base=0, **kw):
    vocab, ops = op_script(seed, **kw)
    py, orc = PyIndex(id_base), pt.Oracle(id_base)
    for op in ops:
        if op[0] == "append":
            _, rows, counted, v = op
            py.append(rows, counted, v)
            orc.append(cdb.sparse_csr(rows), v, counted)
        else:
            _, dels, v = op
            py.delete(dels, v)
            orc.delete(dels, v)
    return vocab, py, orc


@pytest.mark.parametrize("seed", range(40))
def test_heap_mode_equals_the_python_restatement(seed):
    vocab, py, orc = run_script(seed, id_base=seed * 1000)
    df, idf, n = orc.term_stats(vocab)
    assert n == py.n
    for h, d, f in zip(vocab.tolist(), df, idf):
        want_df = len(py.terms[h]) if h in py.terms else 0
        assert d == want_df
        if h in py.terms:
            assert bits(f) == bits(get_idf(py.n, want_df))
        else:
            assert np.isnan(f)
    qs = random_queries(np.random.default_rng(seed + 100), vocab, 30)
    for k in (0, 1, 7, 600):
        ids, scores, counts, panic = orc.search(query_csr(qs), k, "heap")
        for i, q in enumerate(qs):
            try:
                want = py.search_bm25(q, k)
            except Unreachable:
                assert panic[i]
                continue
            assert not panic[i]
            assert counts[i] == len(want)
            assert ids[i, :counts[i]].tolist() == [d for d, _ in want]
            assert [bits(s) for s in scores[i, :counts[i]]] == [bits(s) for _, s in want]
            assert np.all(ids[i, counts[i]:] == 0xFFFFFFFF) and np.all(scores[i, counts[i]:] == 0)


def gamma(m):
    u = 2.0 ** -24
    return m * u / (1 - m * u)


@pytest.mark.parametrize("seed", range(20))
def test_query_and_heap_orders(seed):
    """bit-equal on docs matching <= 2 query terms; with more, each order is within gamma_{m-1} * sum|products| of the exact
    sum (so within twice that of each other)"""
    vocab, ops = op_script(seed, steps=8, vocab_size=8, rows_per_step=60, special=0.0)
    orc, rows = pt.Oracle(), []
    for op in ops:
        if op[0] == "append":
            orc.append(cdb.sparse_csr(op[1]), op[3], op[2])
            rows += op[1]
        else:
            orc.delete(op[1], op[2])
    rng = np.random.default_rng(seed)
    checked = 0
    for q in random_queries(rng, vocab, 20, max_terms=8, absent=0.0):
        a, ta, ma, sa, pa = orc.scores(q, "query")
        b, tb, mb, sb, pb = orc.scores(q, "heap")
        if pb:
            continue
        assert np.array_equal(ta, tb) and np.array_equal(ma, mb)
        few = ta & (ma <= 2)
        assert np.array_equal(a[few].view(np.uint32), b[few].view(np.uint32))
        _, idf, _ = orc.term_stats(np.array(q, np.uint32))
        for r in np.flatnonzero(ta & (ma > 2)):
            pairs = dict(rows[int(r)])
            exact = sum(Fraction(float(f32(f32(pairs[h]) * f))) for h, f in zip(q, idf) if h in pairs)
            bound = gamma(int(ma[r]) - 1) * sa[r]
            assert abs(Fraction(float(a[r])) - exact) <= bound and abs(Fraction(float(b[r])) - exact) <= bound
            checked += 1
    assert checked


def test_summation_orders_really_differ():
    """a seeded case where the reference's heap order and the caller's query order round differently: the GPU contract's
    caveat is not hypothetical"""
    found = 0
    for seed in range(200):
        vocab, ops = op_script(seed, steps=4, vocab_size=6, rows_per_step=40, special=0.0)
        orc = pt.Oracle()
        for op in ops:
            if op[0] == "append":
                orc.append(cdb.sparse_csr(op[1]), op[3], op[2])
            else:
                orc.delete(op[1], op[2])
        q = vocab[::-1].tolist()
        a, ta, ma, _, _ = orc.scores(q, "query")
        b, tb, _, _, pb = orc.scores(q, "heap")
        if pb:
            continue
        diff = ta & (a.view(np.uint32) != b.view(np.uint32))
        assert np.all(ma[diff] > 2)
        found += int(diff.sum())
        if found:
            break
    assert found


def test_df_wraps_past_n_after_cross_version_deletes():
    orc = pt.Oracle()
    rows = [[(7, 1.0), (9, 0.5)], [(7, 2.0)], [(7, 0.25)]]
    orc.append(cdb.sparse_csr(rows), 1)
    df, idf, n = orc.term_stats([7, 9])
    assert n == 3 and df.tolist() == [3, 1]
    orc.delete([0, 1], 2)              # later version: the entries stay (marked) and a tombstone each joins: df 3 -> 5
    df, idf, n = orc.term_stats([7, 9])
    assert n == 1 and df.tolist() == [5, 2]
    # (1 - 5) wraps to 4294967292, which rounds to 4294967296.0 as f32
    want = f32(_libm.log1pf(float(f32(f32(4294967296.0) + f32(0.5)) / f32(5.5))))
    assert bits(idf[0]) == bits(want) == bits(get_idf(1, 5))
    assert idf[0] > 20
    orc.append(cdb.sparse_csr([[(7, 1.0)]]), 2)
    orc.delete([3], 2)                 # same version as its insert: the entry goes, df - 1
    df, _, n = orc.term_stats([7])
    assert n == 1 and df.tolist() == [5]
    orc.delete([3], 2)                 # deleting again changes nothing (the reference would decrement N again)
    assert orc.term_stats([7])[2] == 1
    ids, scores, counts, _ = orc.search(query_csr([[7]]), 0)
    assert ids[0, :counts[0]].tolist() == [2]
    assert bits(scores[0, 0]) == bits(f32(f32(0.25) * idf[0]))


def test_uncounted_rows_and_same_version_delete_of_an_uncounted_row():
    orc = pt.Oracle(id_base=5)
    orc.append(cdb.sparse_csr([[(1, 1.0)], [], [(1, 0.5)]]), 3, np.array([1, 0, 1], np.uint8))
    assert orc.term_stats([1])[2] == 2
    orc.delete([1], 3)
    df, _, n = orc.term_stats([1])
    assert n == 2 and df.tolist() == [2]


def u64_to_f32_exact(x):
    """round-to-nearest-even of the integer x to f32, by exhaustive neighbour comparison in rationals"""
    c = np.float32(float(x))
    best = None
    for cand in (np.nextafter(c, np.float32(0)), c, np.nextafter(c, np.float32(np.inf))):
        d = abs(Fraction(float(cand)) - x)
        if best is None or d < best[0] or (d == best[0] and bits(cand) % 2 == 0):
            best = (d, cand)
    return best[1]


def test_bm25_helpers_equal_the_elementwise_restatement():
    rng = np.random.default_rng(5)
    count = rng.integers(0, 50, 2000).astype(np.uint32)
    count[:4] = [0, 1, 0xFFFFFFFF, 16777217]
    dl = rng.integers(0, 5000, 2000).astype(np.uint32)
    dl[:4] = [0, 0xFFFFFFFF, 33554435, 1]
    for avgdl, k1, b in ((57.3, 1.2, 0.75), (1.0, 1.5, 0.0), (0.0, 1.2, 1.0), (123.456, 0.9, 0.4)):
        got = cdb.bm25_term_frequency(count, dl, avgdl, k1, b)
        with np.errstate(all="ignore"):
            for i in range(count.size):
                c, d = u64_to_f32_exact(int(count[i])), u64_to_f32_exact(int(dl[i]))
                k1f, bf, af = f32(k1), f32(b), f32(avgdl)
                num = f32(c * f32(k1f + f32(1.0)))
                inner = f32(f32(f32(1.0) - bf) + f32(bf * f32(d / af)))
                want = f32(num / f32(c + f32(k1f * inner)))
                assert bits(got[i]) == bits(want), (i, count[i], dl[i], avgdl, k1, b)
    for total, n in ((0, 0), (123, 7), ((1 << 53) + 3, 1), ((1 << 60) + (1 << 36) + 1, 3), (2 ** 64 - 1, 0xFFFFFFFF), (999_999_999, 17)):
        with np.errstate(all="ignore"):
            want = f32(u64_to_f32_exact(total) / u64_to_f32_exact(n))
        got = cdb.average_document_length(total, n)
        assert bits(got) == bits(want), (total, n)


def test_no_cpu_fallback_without_device():
    if cdb.device_count() > 0:
        pytest.skip("CUDA device present")
    with pytest.raises(cdb.CosdataError) as e:
        cdb.TfIdfIndex(capacity_rows=8, capacity_pairs=8)
    assert e.value.status == cdb.Status.CUDA_ERROR


def test_an_exhausted_head_among_others_is_where_the_reference_panics():
    """every entry of term 7 deleted: the reference's heap compares its empty head (unreachable!); the oracle leaves it out,
    flags the query, and the query order scores the other term alone"""
    py, orc = PyIndex(), pt.Oracle()
    rows = [[(7, 1.0), (8, 2.0)], [(8, 0.5)]]
    py.append(rows, [1, 1], 1)
    orc.append(cdb.sparse_csr(rows), 1)
    py.delete([0], 2)
    orc.delete([0], 2)
    with pytest.raises(Unreachable):
        py.search_bm25([7, 8], 0)
    assert py.search_bm25([7], 0) == []          # alone, the empty head is popped and skipped
    _, _, counts, panic = orc.search(query_csr([[7, 8], [7], [8, 7]]), 0, "heap")
    assert panic.tolist() == [True, False, True] and counts[1] == 0
    ids, scores, counts, panic = orc.search(query_csr([[7, 8]]), 0, "query")
    want = py.search_bm25([8], 0)
    assert ids[0, :counts[0]].tolist() == [d for d, _ in want]
    assert [bits(x) for x in scores[0, :counts[0]]] == [bits(x) for _, x in want]
