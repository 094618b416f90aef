"""cdb_tfidf_index_load_files on the GPU: an index loaded from the reference's files equals, bit for bit in ids, counts,
score bits, df, idf bits and N, a GPU index fed the same appends and deletes and the CPU oracle -- before and after further
writes -- and, for the quirk of serialize, a scorer over the deserialized lists.  Also: production scale, tile-boundary
row counts, the capacity_pairs refusal, the counted mask and shard groups with one shard carrying the statistics."""
import numpy as np
import pytest

import cosdata_b200 as cdb
from tests import pytfidf as pt
from tests import tfidf_files as tff
from tests.tfidf_data import query_csr, random_queries, random_rows, zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu

KS = (1, 10, 512, 0)


def assert_equal_search(x, y, queries):
    for k in KS:
        ix, sx, cx = x.batch_search(queries, k)
        iy, sy, cy = y.batch_search(queries, k)
        assert np.array_equal(cx, cy), k
        assert np.array_equal(ix, iy), k
        assert np.array_equal(sx.view(np.uint32), sy.view(np.uint32)), k


def assert_equal_stats(x, y, hashes):
    dx, ix, nx = x.term_stats(hashes)
    dy, iy, ny = y.term_stats(hashes)
    assert nx == ny
    assert np.array_equal(dx, dy)
    assert np.array_equal(ix.view(np.uint32), iy.view(np.uint32))


def replay(ops, ix, orc=None):
    for op in ops:
        if op[0] == "append":
            _, rows, counted, v = op
            if rows:
                ix.append(rows, v, counted)
                if orc is not None:
                    orc.append(_csr(rows), v, counted)
        else:
            _, ids, v = op
            ix.delete_embedding(ids, v)
            if orc is not None:
                orc.delete(ids, v)


def _csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows])
    hs = np.array([h for r in rows for h, _ in r], np.uint32)
    tf = np.array([t for r in rows for _, t in r], np.float32)
    return off, hs, tf


def oracle_search(orc, queries, k):
    o, h = query_csr(queries)
    nq = len(queries)
    kout = 512 if k == 0 or k > 512 else k
    ids = np.zeros((nq, kout), np.uint32)
    sc = np.zeros((nq, kout), np.float32)
    cnt = np.zeros(nq, np.uint32)
    pt.lib().to_search(orc.h, pt.MODES["query"], pt._p(o), pt._p(h), nq, k, pt._p(ids), pt._p(sc), pt._p(cnt), None)
    return ids, sc, cnt


def assert_oracle(x, orc, queries):
    for k in KS:
        ix, sx, cx = x.batch_search(queries, k)
        wi, ws, wc = oracle_search(orc, queries, k)
        assert np.array_equal(cx, wc), k
        assert np.array_equal(ix, wi), k
        assert np.array_equal(sx.view(np.uint32), ws.view(np.uint32)), k


@pytest.mark.parametrize("seed", range(4))
def test_loaded_index_equals_the_same_history_and_the_oracle(seed, tmp_path):
    hist, ops, vocab = tff.seeded_history(seed, n_versions=5, docs_per_version=60, vocab_size=14,
                                          flush_after={2, 4} if seed % 2 else None)
    d = str(tmp_path / "tf")
    hist.save(d)
    n = sum(len(op[1]) for op in ops if op[0] == "append")
    counted = np.array([1 if c else 0 for op in ops if op[0] == "append" for c in op[2]], np.uint8)
    fresh = cdb.TfIdfIndex(capacity_rows=4 * n + 64, capacity_pairs=1 << 16)
    orc = pt.Oracle()
    replay(ops, fresh, orc)
    ld = cdb.TfIdfIndex(capacity_rows=4 * n + 64, capacity_pairs=1 << 16)
    with cdb.TfIdfFiles(d) as f:
        # the mask names the documents with text that are still live: stopword-only documents keep counting
        mask = counted.copy()
        mask[sorted(hist.deleted)] = 0
        ld.load_files(f, n, counted=mask)
    assert len(ld) == n
    rng = np.random.default_rng(seed + 100)
    qs = random_queries(rng, vocab, 40)
    hashes = np.concatenate([vocab, rng.integers(0, 1 << 32, 8, dtype=np.uint64).astype(np.uint32)])
    assert_equal_stats(ld, fresh, hashes)
    assert_equal_search(ld, fresh, qs)
    assert_oracle(ld, orc, qs)
    # rows deleted before the files were written come back empty and not deleted: deleted_rows differs, results do not
    dl, tl = ld.deleted_rows()
    df_, tf_ = fresh.deleted_rows()
    assert tl == 0 and tf_ == len(hist.deleted)
    # more writes on both: appends and deletes in the files' last version and later, on loaded and on new rows
    last = max(op[-1] for op in ops)
    more_rows, more_counted = random_rows(rng, 50, vocab)
    later = [("append", more_rows[:25], more_counted[:25], last),
             ("delete", rng.choice(n + 25, 20).astype(np.uint32), last),
             ("append", more_rows[25:], more_counted[25:], last + 1),
             ("delete", rng.choice(n + 50, 30).astype(np.uint32), last + 2)]
    for op in later:
        replay([op], fresh, orc)
        replay([op], ld)
        assert_equal_stats(ld, fresh, hashes)
        assert_equal_search(ld, fresh, qs)
        assert_oracle(ld, orc, qs)
    for x in (fresh, ld, orc):
        x.close()


def test_quirk_file_loads_as_deserialize_reads_it(tmp_path):
    rng = np.random.default_rng(5)
    vocab = rng.choice(1 << 31, 10, replace=False).astype(np.uint32)
    h = tff.History()
    rows, counted = random_rows(rng, 80, vocab, uncounted=0.0)
    for r, row in enumerate(rows):
        h.insert(r, row, 1)
    h.flush()
    for r in range(0, 80, 7):
        h.delete(r, 1)          # in the insert's version after the flush: live again after a reload
    more, _ = random_rows(rng, 40, vocab, uncounted=0.0)
    for r, row in enumerate(more):
        h.insert(80 + r, row, 2)
    for r in range(3, 120, 11):
        h.delete(r, 2)
    h.flush()
    d = str(tmp_path / "tf")
    h.save(d)
    n_docs, terms = tff.deserialize(*tff.read_dir(d))
    assert terms != h.root.terms()
    ld = cdb.TfIdfIndex(capacity_rows=256, capacity_pairs=4096)
    with cdb.TfIdfFiles(d) as f:
        ld.load_files(f, 120)
    df, _, n = ld.term_stats(vocab)
    assert n == n_docs and df.tolist() == [terms[int(x)][0] for x in vocab]
    qs = random_queries(rng, vocab, 30, absent=0.0)
    for k in KS:
        gi, gs, gc = ld.batch_search(qs, k)
        wi, ws, wc = tff.search_lists(n_docs, terms, qs, k)
        assert np.array_equal(gc, wc) and np.array_equal(gi, wi) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), k
    ld.close()


def bulk_files(tmp_path, n, seed, vocab):
    off, hs, tf = zipf_docs(seed, n, vocab=vocab)
    n1 = (2 * n) // 3
    dele = np.sort(np.random.default_rng(seed).choice(n1, max(1, n // 100), replace=False))
    d = str(tmp_path / f"bulk{n}_{seed}")
    tff.write_bulk(d, off, hs, tf, n1, dele)
    return d, off, hs, tf, n1, dele


def bulk(tmp_path, n, seed=1, vocab=1_000_000):
    """files of n documents in two versions with 1 % deleted in the second, and the GPU index of the same history"""
    d, off, hs, tf, n1, dele = bulk_files(tmp_path, n, seed, vocab)
    fresh = cdb.TfIdfIndex(capacity_rows=n + 1, capacity_pairs=len(hs) + 64)
    fresh.append((off[:n1 + 1], hs[:int(off[n1])], tf[:int(off[n1])]), 1)
    fresh.append((off[n1:] - off[n1], hs[int(off[n1]):], tf[int(off[n1]):]), 2)
    fresh.delete_embedding(dele, 2)
    mask = np.ones(n, np.uint8)
    mask[dele] = 0
    return d, fresh, mask, hs


@pytest.mark.parametrize("n", [(1 << 15) - 1, (1 << 15) + 1, 1 << 16])
def test_tile_boundaries_and_the_capacity_refusal(n, tmp_path):
    d, fresh, mask, hs = bulk(tmp_path, n, seed=n, vocab=20_000)
    big = bulk_files(tmp_path, 2 * n, n + 1, 20_000)[0]
    with cdb.TfIdfFiles(d) as f, cdb.TfIdfFiles(big) as fb:
        live = f.info["live"]
        assert fb.info["live"] > live
        # more live pairs than capacity_pairs: refused, and the same handle then loads files that fit
        ld = cdb.TfIdfIndex(capacity_rows=2 * n + 1, capacity_pairs=live)
        with pytest.raises(cdb.CosdataError) as e:
            ld.load_files(fb, 2 * n)
        assert e.value.status == cdb.Status.INVALID_PARAMS
        assert len(ld) == 0
        ld.load_files(f, n, counted=mask)
    assert len(ld) == n
    qs = zipf_queries(9, 64, vocab=20_000)
    assert_equal_search(ld, fresh, qs)
    assert_equal_stats(ld, fresh, np.unique(hs)[:5000])
    fresh.close()
    ld.close()


def test_production_scale(tmp_path):
    n = 1_000_000
    d, fresh, mask, hs = bulk(tmp_path, n)
    ld = cdb.TfIdfIndex(capacity_rows=n + 1, capacity_pairs=len(hs) + 64)
    with cdb.TfIdfFiles(d) as f:
        ld.load_files(f, n, counted=mask)
    qs = zipf_queries(11, 64)
    assert_equal_search(ld, fresh, qs)
    assert_equal_stats(ld, fresh, np.unique(hs)[::50])
    # a loaded index is not empty: a second load into it is refused
    with cdb.TfIdfFiles(d) as f:
        with pytest.raises(cdb.CosdataError):
            ld.load_files(f, n)
    fresh.close()
    ld.close()


def test_counted_mask_stopword_document_deleted_lowers_n(tmp_path):
    h = tff.History()
    h.insert(0, [(0x10001, 1.0)], 1)
    h.insert(1, [], 1)                       # text of stopwords only: no pair, but it counts
    h.insert(2, [(0x10001, 2.0), (0x20001, 1.0)], 1)
    h.flush()
    d = str(tmp_path / "tf")
    h.save(d)
    ld = cdb.TfIdfIndex(capacity_rows=8, capacity_pairs=64)
    with cdb.TfIdfFiles(d) as f:
        with pytest.raises(cdb.CosdataError):
            ld.load_files(f, 3, counted=np.array([0, 1, 1], np.uint8))    # a 0 on a row with live words
        assert len(ld) == 0
        ld.load_files(f, 3, counted=np.array([1, 1, 1], np.uint8))
    assert ld.term_stats([0x10001])[2] == 3
    ld.delete_embedding([1], 2)
    assert ld.term_stats([0x10001])[2] == 2
    fresh = cdb.TfIdfIndex(capacity_rows=8, capacity_pairs=64)
    fresh.append([[(0x10001, 1.0)], [], [(0x10001, 2.0), (0x20001, 1.0)]], 1)
    fresh.delete_embedding([1], 2)
    assert_equal_stats(ld, fresh, [0x10001, 0x20001])
    assert_equal_search(ld, fresh, [[0x10001], [0x20001, 0x10001]])


def device_search(g, qs, k):
    """cdb_tfidf_search_batch_sharded_device on torch buffers"""
    import torch
    o, h = query_csr(qs)
    nq, kout = len(qs), 512 if k == 0 or k > 512 else k
    dev = torch.device("cuda", 0)
    do = torch.from_numpy(o.view(np.int64)).to(dev)
    dh = torch.from_numpy(np.ascontiguousarray(h).view(np.int32)).to(dev)
    ids = torch.zeros((nq, kout), dtype=torch.int32, device=dev)
    sc = torch.zeros((nq, kout), dtype=torch.float32, device=dev)
    cnt = torch.zeros(nq, dtype=torch.int32, device=dev)
    g.search_tfidf_device(do.data_ptr(), dh.data_ptr(), nq, int(o[-1]), k, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr())
    torch.cuda.synchronize()
    return ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)


def test_shard_group_with_one_carrying_slot(tmp_path):
    from cosdata_b200.sharding import ShardGroup
    hist, ops, vocab = tff.seeded_history(21, n_versions=4, docs_per_version=80, vocab_size=16)
    d = str(tmp_path / "tf")
    hist.save(d)
    n = sum(len(op[1]) for op in ops if op[0] == "append")
    counted = np.array([1 if c else 0 for op in ops if op[0] == "append" for c in op[2]], np.uint8)
    mask = counted.copy()
    mask[sorted(hist.deleted)] = 0
    cap = 2 * n + 64
    half = n // 2
    whole = cdb.TfIdfIndex(capacity_rows=cap, capacity_pairs=1 << 16)
    s0 = cdb.TfIdfIndex(capacity_rows=half, capacity_pairs=1 << 16, id_base=0)
    s1 = cdb.TfIdfIndex(capacity_rows=cap - half, capacity_pairs=1 << 16, id_base=half)
    with cdb.TfIdfFiles(d) as f:
        whole.load_files(f, n, counted=mask)
        s0.load_files(f, half, counted=mask[:half], carry_stats=True)
        s1.load_files(f, n - half, counted=mask[half:], carry_stats=False)
    g = ShardGroup.local([0, 0])
    g.attach_tfidf(0, s0)
    g.attach_tfidf(1, s1)
    rng = np.random.default_rng(3)
    qs = random_queries(rng, vocab, 48)

    def check():
        for k in KS:
            wi, ws, wc = whole.batch_search(qs, k)
            for gi, gs, gc in (g.search_tfidf(qs, k), device_search(g, qs, k)):
                assert np.array_equal(gc, wc) and np.array_equal(gi, wi) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), k
    check()
    # deletes in the insert's version of shard 1's rows of the files' last version: each removes its entries (df - 1), so
    # shard 1, loaded with df 0, goes below zero mod 2^32, and the group's wrapping sums still equal the whole index
    last = max(op[-1] for op in ops)
    last_rows = next(op[1] for op in reversed(ops) if op[0] == "append" and op[3] == last)
    same = np.array([r for r in range(n - len(last_rows), n)
                     if r >= half and r not in hist.deleted and hist.docs[r][1] and hist.docs[r][0]], np.uint32)
    assert same.size >= 3
    whole.delete_embedding(same, last)
    s1.delete_embedding(same - half, last)
    d0, _, n0 = s0.term_stats(vocab)
    d1, _, n1 = s1.term_stats(vocab)
    dw, _, nw = whole.term_stats(vocab)
    assert (d1 >= 1 << 31).any(), "no df of shard 1 went below zero"
    assert np.array_equal((d0.astype(np.uint64) + d1) % (1 << 32), dw) and (n0 + n1) % (1 << 32) == nw
    check()
    # later writes on both shards
    del0 = np.arange(0, half, 3, dtype=np.uint32)
    del1 = np.arange(half, n, 2, dtype=np.uint32)
    whole.delete_embedding(np.concatenate([del0, del1]), last + 1)
    s0.delete_embedding(del0, last + 1)
    s1.delete_embedding(del1 - half, last + 1)
    rows, rc = random_rows(rng, 30, vocab)
    whole.append(rows, last + 1, rc)
    # the group's rows past n go to shard 1 (whole index rows n.. = ids n..)
    s1.append(rows, last + 1, rc)
    check()
    g.close()
    for x in (whole, s0, s1):
        x.close()
