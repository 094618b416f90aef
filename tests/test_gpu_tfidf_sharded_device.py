"""The sharded TF-IDF search from device buffers (cdb_tfidf_search_batch_sharded_device, csrc/shard_group.cu), with the
group's idf computed on the device, and the single index's idf refresh on the device (bm25_idf.h).

The device form must return the host form's ids, counts and score bits, and so one index's over every shard's rows, on a
per-rank group of world 1, a one-slot local group and loopback groups of 2 and 3 slots on device 0; both forms run one
plan, so both launch the same kernels.  The shards see
appends in several versions, deletes in the insert's version and later ones (df > N), an empty shard, hashes some or all
shards never saw, repeated hashes, a query of more than 512 terms, every k class and a batch of two group chunks.  The
launch plan, the asynchrony on the caller's stream and the refusals that need the group are pinned here too."""
import numpy as np
import pytest

import cosdata_b200 as cdb
from cosdata_b200.sharding import ShardGroup
from tests import pytfidf as pt
from tests import text_plan as tp
from tests.tfidf_data import query_csr, random_rows

pytestmark = pytest.mark.gpu

KS = (0, 1, 10, 512, 600)


def device_launches(nq, shard_rows, n_hashes):
    """kernel launches of one call, host or device form, on the one-slot and loopback groups here"""
    return tp.tfidf_group_search_launches(nq, [tp.n_tiles(r) for r in shard_rows], n_hashes, loopback=True)


def kout(k):
    return 512 if k == 0 or k > 512 else k


class Layout:
    """shards over global id ranges [bounds[r], bounds[r+1]) in a group of the named kind, next to one whole index; appends
    and deletes go to both with the same versions"""

    def __init__(self, kind, bounds):
        n = len(bounds) - 1
        self.kind, self.bounds = kind, bounds
        self.g = ShardGroup.rank(None, 1, 0, 0) if kind == "rank" else ShardGroup.local([0] * n)
        assert kind != "rank" or n == 1
        self.parts = []
        for r in range(n):
            ix = cdb.TfIdfIndex(capacity_rows=bounds[r + 1] - bounds[r], capacity_pairs=1 << 16, id_base=bounds[r], device=0)
            self.g.attach_tfidf(r, ix)
            self.parts.append(ix)
        self.whole = cdb.TfIdfIndex(capacity_rows=bounds[-1], capacity_pairs=1 << 18)
        self.n = 0

    def append(self, rows, counted, version):
        counted = np.asarray(counted, np.uint8)
        self.whole.append(rows, version, counted)
        for r, ix in enumerate(self.parts):
            a, b = max(self.n, self.bounds[r]), min(self.n + len(rows), self.bounds[r + 1])
            if a < b:
                ix.append(rows[a - self.n:b - self.n], version, counted[a - self.n:b - self.n])
        self.n += len(rows)

    def delete(self, rows, version):
        rows = np.asarray(rows, np.uint32)
        self.whole.delete_embedding(rows, version)
        for r, ix in enumerate(self.parts):
            mine = rows[(rows >= self.bounds[r]) & (rows < self.bounds[r + 1])]
            if mine.size:
                ix.delete_embedding(mine - self.bounds[r], version)

    def shard_rows(self):
        return [max(0, min(self.n, self.bounds[r + 1]) - self.bounds[r]) for r in range(len(self.parts))]

    def close(self):
        self.g.close()
        for x in self.parts + [self.whole]:
            x.close()


def to_device(qs):
    import torch
    o, h = query_csr(qs)
    dev = torch.device("cuda", 0)
    d_o = torch.from_numpy(o.astype(np.int64)).to(dev)
    d_h = torch.from_numpy(h.view(np.int32) if h.size else np.zeros(1, np.int32)).to(dev)
    return d_o, d_h, len(qs), int(h.size)


def outputs(nq, k):
    import torch
    dev = torch.device("cuda", 0)
    ids = torch.full((max(nq, 1), kout(k)), 0x5A5A5A5A, dtype=torch.int32, device=dev)
    scores = torch.full((max(nq, 1), kout(k)), float("nan"), dtype=torch.float32, device=dev)
    counts = torch.full((max(nq, 1),), 0x5A5A5A5A, dtype=torch.int32, device=dev)
    return ids, scores, counts


def device_search(g, qs, k, stream=None):
    """the device form on a torch stream (the current one by default), results read back after synchronising"""
    import torch
    d_o, d_h, nq, nh = to_device(qs)
    ids, scores, counts = outputs(nq, k)
    s = stream or torch.cuda.current_stream(torch.device("cuda", 0))
    g.search_tfidf_device(d_o.data_ptr(), d_h.data_ptr(), nq, nh, k, ids.data_ptr(), scores.data_ptr(), counts.data_ptr(),
                          s.cuda_stream)
    s.synchronize()
    return (ids.cpu().numpy().view(np.uint32)[:nq], scores.cpu().numpy()[:nq], counts.cpu().numpy().view(np.uint32)[:nq])


def check(got, want):
    ids, scores, counts = got
    w_ids, w_scores, w_counts = want[:3]
    assert np.array_equal(counts, w_counts)
    assert np.array_equal(ids, w_ids)
    assert np.array_equal(np.ascontiguousarray(scores).view(np.uint32), np.ascontiguousarray(w_scores).view(np.uint32))


def corpus_script(seed, vocab):
    """appends in versions 1, 2 and 4, deletes in the insert's version and in later ones, on 300 rows; vocab[0] is in
    every counted row, so its df passes N once later-version deletes have run; vocab[1] only in rows below 100"""
    rng = np.random.default_rng(seed)
    rows, counted = random_rows(rng, 300, vocab[2:], max_terms=5)
    for r in range(300):
        if counted[r]:
            rows[r] = [(int(vocab[0]), 0.75 + 0.01 * (r % 7))] + rows[r]
            if r < 100 and r % 3 == 0:
                rows[r] = rows[r] + [(int(vocab[1]), 1.25)]
    return [("append", rows[:100], counted[:100], 1),
            ("append", rows[100:220], counted[100:220], 2),
            ("delete", [101, 150, 219, 205], 2),                 # the insert's version: df - 1
            ("delete", rng.choice(220, 60, replace=False), 3),   # later: df + 1, N - 1
            ("append", rows[220:], counted[220:], 4),
            ("delete", [230, 5, 240], 4)]


def queries(seed, vocab, nq=40):
    rng = np.random.default_rng(seed)
    qs = []
    for i in range(nq):
        m = int(rng.integers(0, 9))
        q = rng.choice(vocab, m).tolist()
        q = [int(rng.integers(1 << 31, 1 << 32)) if rng.random() < 0.1 else int(h) for h in q]
        qs.append(q)
    qs += [[], [int(vocab[0]), int(vocab[0]), int(vocab[2])], [int(vocab[1])], [0xFFFFFFFE, 0xFFFFFFFF],
           rng.choice(vocab, 700).tolist()]   # the last: more than 512 terms, with repeats
    return qs


LAYOUTS = [("rank", [0, 400]), ("local", [0, 400]), ("loop", [0, 200, 400]), ("loop", [0, 150, 300, 400])]


@pytest.mark.parametrize("kind,bounds", LAYOUTS, ids=["rank1", "local1", "loop2", "loop3_empty"])
def test_device_form_equals_host_form_and_whole_index(kind, bounds):
    import torch
    vocab = np.random.default_rng(5).choice(1 << 31, 40, replace=False).astype(np.uint32)
    lay = Layout(kind, bounds)
    qs = queries(11, vocab)
    o, h = query_csr(qs)
    for i, op in enumerate(corpus_script(3, vocab)):
        if op[0] == "append":
            lay.append(op[1], op[2], op[3])
        else:
            lay.delete(op[1], op[2])
        if i in (1, 3, 5):
            for k in KS:
                before = cdb.kernel_launch_count()
                got = device_search(lay.g, qs, k)
                assert cdb.kernel_launch_count() - before == device_launches(len(qs), lay.shard_rows(), h.size)
                before = cdb.kernel_launch_count()
                host = lay.g.search_tfidf(qs, k)
                assert cdb.kernel_launch_count() - before == device_launches(len(qs), lay.shard_rows(), h.size)
                check(got, host)
                check(got, lay.whole.batch_search(qs, k))
    # vocab[0]: df past N in the whole index after the later-version deletes
    df, _, n_docs = lay.whole.term_stats(vocab[:1])
    assert df[0] > n_docs
    if bounds[-2] == 300:
        assert lay.shard_rows()[-1] == 0                 # the empty shard
    # nothing is launched for an empty batch
    before = cdb.kernel_launch_count()
    z = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    lay.g.search_tfidf_device(z.data_ptr(), z.data_ptr(), 0, 0, 10, z.data_ptr(), z.data_ptr(), z.data_ptr(), None)
    torch.cuda.synchronize()
    assert cdb.kernel_launch_count() == before
    lay.close()


def test_device_form_over_two_group_chunks():
    """3 loopback slots: a group chunk is 256 MB / (3 * 4096) = 21845 queries, so 21850 queries take two"""
    vocab = np.random.default_rng(6).choice(1 << 31, 30, replace=False).astype(np.uint32)
    lay = Layout("loop", [0, 150, 300, 400])
    for op in corpus_script(4, vocab):
        if op[0] == "append":
            lay.append(op[1], op[2], op[3])
        else:
            lay.delete(op[1], op[2])
    base = queries(12, vocab, nq=45)
    qs = (base * (21850 // len(base) + 1))[:21850]
    assert len(tp.chunks(len(qs), tp.group_chunk(len(qs), 3, tp.TF_BUCKETS * 8))) == 2
    o, h = query_csr(qs)
    for k in (10, 0):
        before = cdb.kernel_launch_count()
        got = device_search(lay.g, qs, k)
        assert cdb.kernel_launch_count() - before == device_launches(len(qs), lay.shard_rows(), h.size)
        before = cdb.kernel_launch_count()
        host = lay.g.search_tfidf(qs, k)
        assert cdb.kernel_launch_count() - before == device_launches(len(qs), lay.shard_rows(), h.size)
        check(got, host)
        check(got, lay.whole.batch_search(qs, k))
    lay.close()


@pytest.mark.parametrize("kind,bounds", [("rank", [0, 400]), ("loop", [0, 200, 400])], ids=["rank1", "loop2"])
def test_device_form_is_asynchronous_on_the_callers_stream(kind, bounds):
    import torch
    vocab = np.random.default_rng(7).choice(1 << 31, 30, replace=False).astype(np.uint32)
    lay = Layout(kind, bounds)
    for op in corpus_script(5, vocab):
        if op[0] == "append":
            lay.append(op[1], op[2], op[3])
        else:
            lay.delete(op[1], op[2])
    qs = queries(13, vocab)
    want = lay.g.search_tfidf(qs, 10)
    dev = torch.device("cuda", 0)
    s = torch.cuda.Stream(dev)
    check(device_search(lay.g, qs, 10, stream=s), want)   # the group's buffers are sized: no allocation below
    d_o, d_h, nq, nh = to_device(qs)
    ids, scores, counts = outputs(nq, 10)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)                        # ~0.5 s of the caller's earlier work
    lay.g.search_tfidf_device(d_o.data_ptr(), d_h.data_ptr(), nq, nh, 10, ids.data_ptr(), scores.data_ptr(), counts.data_ptr(),
                              s.cuda_stream)
    ev = torch.cuda.Event()
    ev.record(s)
    assert not ev.query(), "the call waited for the device"
    ev.synchronize()
    check((ids.cpu().numpy().view(np.uint32), scores.cpu().numpy(), counts.cpu().numpy().view(np.uint32)), want)
    lay.close()


def test_refusals_that_need_the_group():
    import torch
    z = torch.zeros(4, dtype=torch.int64, device="cuda:0")
    g = ShardGroup.local([0, 0])
    t = cdb.TfIdfIndex(capacity_rows=10, capacity_pairs=10, device=0)
    g.attach_tfidf(0, t)
    with pytest.raises(cdb.CosdataError, match="no tf-idf shard"):   # slot 1 has none
        g.search_tfidf_device(z.data_ptr(), z.data_ptr(), 1, 0, 10, z.data_ptr(), z.data_ptr(), z.data_ptr())
    g.close()
    t.close()
    if cdb.device_count() < 2:
        pytest.skip("a local group on two devices needs two GPUs")
    g = ShardGroup.local([0, 1])
    a = cdb.TfIdfIndex(capacity_rows=10, capacity_pairs=10, device=0)
    b = cdb.TfIdfIndex(capacity_rows=10, capacity_pairs=10, id_base=10, device=1)
    g.attach_tfidf(0, a)
    g.attach_tfidf(1, b)
    with pytest.raises(cdb.CosdataError, match="share one device"):
        g.search_tfidf_device(z.data_ptr(), z.data_ptr(), 1, 0, 10, z.data_ptr(), z.data_ptr(), z.data_ptr())
    g.close()
    a.close()
    b.close()


def test_device_idf_after_single_index_writes():
    """term j is in rows 0..j (df 1..200 after the appends); later-version deletes push the popular terms' df past N"""
    n = 200
    terms = np.arange(1000, 1000 + n, dtype=np.uint32)
    rows = [[(int(terms[j]), 1.0) for j in range(r, n)] for r in range(n)]
    ix = cdb.TfIdfIndex(capacity_rows=2 * n, capacity_pairs=1 << 16)

    def agrees():
        df, idf, n_docs = ix.term_stats(terms)
        want = np.array([pt.idf(n_docs, int(d)) for d in df], np.float32)
        assert np.array_equal(idf.view(np.uint32), want.view(np.uint32))
        return df, n_docs

    ix.append(rows[:120], 1)
    agrees()
    ix.append(rows[120:], 2)
    df, n_docs = agrees()
    assert df.min() == 1 and df.max() == n == n_docs
    ix.delete_embedding(np.arange(150, 160, dtype=np.uint32), 2)     # the insert's version: df - 1
    agrees()
    ix.delete_embedding(np.arange(0, 90, dtype=np.uint32), 5)        # later: df + 1, N - 1
    df, n_docs = agrees()
    assert df.max() > n_docs
    ix.append([[(int(terms[-1]), 2.0)], []], 6, np.array([1, 0], np.uint8))
    agrees()
    ix.close()
