"""The TF-IDF / BM25 index on the GPU (cdb_tfidf_*) against the CPU oracle's `query` summation order
(tests/tfidf_oracle.c): ids, counts and score bits equal, and N, df and idf bits equal, on tf values of 0, -0, negative, inf
and NaN; empty, uncounted and deleted rows; empty queries, absent and repeated hashes; terms whose every entry is deleted;
bucket and +-0 ties; id_base near 2^32 - 2; k = 1, 10, 512, 0 (None) and 1000; corpora of several row tiles appended in
pieces that end mid-tile with same- and cross-version deletes; batch 1 and 1024, the device twin on a side stream and 8
host threads."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

import cosdata_b200 as cdb
from tests import pytfidf as pt
from tests.sparse_data import concat_csr, slice_csr
from tests.tfidf_data import op_script, query_csr, random_queries, zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu

KS = (1, 10, 512, 0, 1000)


def check(got, want):
    ids, scores, counts = got
    w_ids, w_scores, w_counts = want[:3]
    assert np.array_equal(counts, w_counts)
    assert np.array_equal(ids, w_ids)
    assert np.array_equal(np.ascontiguousarray(scores).view(np.uint32), np.ascontiguousarray(w_scores).view(np.uint32))


def check_stats(ix, orc, hashes):
    got = ix.term_stats(hashes)
    want = orc.term_stats(hashes)
    assert got[2] == want[2]
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))


def both(id_base=0, capacity_rows=1 << 16, capacity_pairs=1 << 20):
    return cdb.TfIdfIndex(capacity_rows=capacity_rows, capacity_pairs=capacity_pairs, id_base=id_base), pt.Oracle(id_base)


@pytest.mark.parametrize("seed", range(12))
def test_op_scripts_against_the_oracle(seed):
    """adversarial tf values, uncounted rows, versioned deletes (some twice), absent and repeated query hashes"""
    id_base = [0, 3, 0xFFFFFFFF - 1 - 400][seed % 3]
    ix, orc = both(id_base, capacity_rows=400, capacity_pairs=4000)
    vocab, ops = op_script(seed, steps=8, vocab_size=12, rows_per_step=40)
    qs = random_queries(np.random.default_rng(seed), vocab, 40) + [[]]
    for op in ops:
        if op[0] == "append":
            ix.append(op[1], op[3], op[2])
            orc.append(cdb.sparse_csr(op[1]), op[3], op[2])
        else:
            ix.delete_embedding(op[1], op[2])
            orc.delete(op[1], op[2])
        check_stats(ix, orc, np.concatenate([vocab, np.array([12345], np.uint32)]))
        for k in KS:
            check(ix.batch_search(qs, k), orc.search(query_csr(qs), k))
    ix.close()


def test_ties_zero_signs_and_empty_lists():
    ix, orc = both(id_base=0xFFFFFFFF - 1 - 2000, capacity_rows=2000)
    rows = []
    for r in range(1500):
        if r % 7 == 0:
            rows.append([(1, 0.0)])
        elif r % 7 == 1:
            rows.append([(1, -0.0)])
        elif r % 7 == 2:
            rows.append([(1, 1.0), (2, 2.0)])
        elif r % 7 == 3:
            rows.append([(2, 2.0), (1, 1.0)])       # the same score as the previous row: a tie in (usually) another bucket
        elif r % 7 == 4:
            rows.append([(3, float("nan")), (1, 1.0)])
        elif r % 7 == 5:
            rows.append([(4, float("-inf"))])
        else:
            rows.append([])
    counted = np.array([0 if (r % 7 == 6 and r % 2) else 1 for r in range(1500)], np.uint8)
    ix.append(rows, 1, counted)
    orc.append(cdb.sparse_csr(rows), 1, counted)
    dead = np.array([r for r in range(1500) if r % 7 == 5], np.uint32)   # every entry of term 4
    ix.delete_embedding(dead, 1)
    orc.delete(dead, 1)
    qs = [[1], [1, 2], [2, 1], [3], [4], [4, 1], [1, 1, 2], [9], [], [1, 4, 3, 2]]
    check_stats(ix, orc, [1, 2, 3, 4, 9])
    for k in KS:
        check(ix.batch_search(qs, k), orc.search(query_csr(qs), k))
    ids, scores, counts = ix.batch_search([[1]], 0)
    live = [r for r in range(1500) if r % 7 < 5]                     # rows holding term 1
    assert counts[0] == len({(ix.desc.id_base + r) % 512 for r in live}) > 500
    ix.close()


def multi_tile(seed, n):
    return zipf_docs(seed, n, vocab=5000, mean_terms=12)


def test_tiles_appended_in_pieces_with_versioned_deletes():
    n = 110_000
    corpus = multi_tile(3, n)
    ix, orc = both(id_base=1000, capacity_rows=n, capacity_pairs=len(corpus[1]))
    qs = zipf_queries(4, 1024, vocab=5000)
    cuts = [0, 30_001, 70_000, 98_304, n]           # tiles hold 32768 rows; pieces end mid-tile and on a boundary
    rng = np.random.default_rng(5)
    version = 2
    for i in range(len(cuts) - 1):
        piece = slice_csr(corpus, cuts[i], cuts[i + 1])
        ix.append(piece, version)
        orc.append(piece, version)
        dels = rng.choice(cuts[i + 1], 300).astype(np.uint32)
        same = dels[dels >= cuts[i]]                 # rows of this append: removed in their own version
        ix.delete_embedding(same, version)
        orc.delete(same, version)
        version += 1
        old = dels[dels < cuts[i]]                   # older rows: marked plus a tombstone
        ix.delete_embedding(old, version)
        orc.delete(old, version)
        check(ix.batch_search(qs[:64], 10), orc.search(query_csr(qs[:64]), 10))
    got_del, total = ix.deleted_rows()
    assert total == int(got_del.sum()) > 0
    check_stats(ix, orc, np.unique(corpus[1])[:2000])
    for k in KS:
        check(ix.batch_search(qs, k), orc.search(query_csr(qs), k))
    check(ix.batch_search(qs[:1], 10), orc.search(query_csr(qs[:1]), 10))
    ix.close()


def test_device_twin_on_a_side_stream_and_threads():
    import torch
    from cosdata_b200 import _lib
    corpus = multi_tile(6, 70_000)
    ix, orc = both(capacity_rows=70_000, capacity_pairs=len(corpus[1]))
    ix.append(corpus, 1)
    orc.append(corpus, 1)
    qs = zipf_queries(7, 1024, vocab=5000)
    want = orc.search(query_csr(qs), 100)
    check(ix.batch_search(qs, 100), want)
    dev = torch.device("cuda", 0)
    qo, qh = query_csr(qs)
    o = torch.from_numpy(qo.astype(np.int64)).to(dev)
    h = torch.from_numpy(qh.astype(np.int32)).to(dev)
    s = torch.cuda.Stream(dev)
    ids = torch.zeros((1024, 100), dtype=torch.int32, device=dev)
    sc = torch.zeros((1024, 100), dtype=torch.float32, device=dev)
    cnt = torch.zeros(1024, dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)
    rc = _lib.load().cdb_tfidf_search_batch_device(ix.h, o.data_ptr(), h.data_ptr(), 1024, 100, ids.data_ptr(), sc.data_ptr(),
                                                    cnt.data_ptr(), C.c_void_p(s.cuda_stream))
    assert rc == 0
    s.synchronize()
    check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), want)
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        for got in ex.map(lambda _: ix.batch_search(qs, 100), range(16)):
            check(got, want)
    ix.close()


def test_append_and_delete_after_queued_device_searches():
    """an append rewrites the last partial tile and every idf; searches already queued see the index as it was"""
    import torch
    from cosdata_b200 import _lib
    corpus = multi_tile(8, 20_000)
    first = slice_csr(corpus, 0, 12_000)
    ix, orc = both(capacity_rows=20_000, capacity_pairs=len(corpus[1]))
    ix.append(first, 1)
    orc.append(first, 1)
    qs = zipf_queries(9, 256, vocab=5000)
    want = orc.search(query_csr(qs), 10)
    dev = torch.device("cuda", 0)
    qo, qh = query_csr(qs)
    o = torch.from_numpy(qo.astype(np.int64)).to(dev)
    h = torch.from_numpy(qh.astype(np.int32)).to(dev)
    s = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    outs = []
    for _ in range(8):
        ids = torch.zeros((256, 10), dtype=torch.int32, device=dev)
        sc = torch.zeros((256, 10), dtype=torch.float32, device=dev)
        cnt = torch.zeros(256, dtype=torch.int32, device=dev)
        assert _lib.load().cdb_tfidf_search_batch_device(ix.h, o.data_ptr(), h.data_ptr(), 256, 10, ids.data_ptr(), sc.data_ptr(),
                                                         cnt.data_ptr(), C.c_void_p(s.cuda_stream)) == 0
        outs.append((ids, sc, cnt))
    rest = slice_csr(corpus, 12_000, 20_000)
    ix.append(rest, 2)
    orc.append(rest, 2)
    ix.delete_embedding(np.arange(0, 20_000, 3, dtype=np.uint32), 2)
    orc.delete(np.arange(0, 20_000, 3, dtype=np.uint32), 2)
    s.synchronize()
    for ids, sc, cnt in outs:
        check((ids.cpu().numpy().view(np.uint32), sc.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)), want)
    check(ix.batch_search(qs, 10), orc.search(query_csr(qs), 10))
    ix.close()


def test_invalid_calls_change_nothing():
    ix, orc = both(capacity_rows=10, capacity_pairs=20)
    ix.append([[(1, 0.5), (2, 1.0)], [(1, 0.25)]], 5)
    orc.append(cdb.sparse_csr([[(1, 0.5), (2, 1.0)], [(1, 0.25)]]), 5)
    for bad in (lambda: ix.append([[(3, 1.0), (3, 2.0)]], 5),                  # a row repeating a hash
                lambda: ix.append([[(3, 1.0)]], 5, counted=[0]),                # an uncounted row with pairs
                lambda: ix.append([[(3, 1.0)]], 4),                             # an older version
                lambda: ix.append([[(3, 1.0)]] * 9, 5),                         # capacity_rows
                lambda: ix.delete_embedding([2], 5),                            # not appended
                lambda: ix.delete_embedding([0], 4)):                           # an older version
        with pytest.raises(cdb.CosdataError) as e:
            bad()
        assert e.value.status == cdb.Status.INVALID_PARAMS
    assert len(ix) == 2
    check_stats(ix, orc, [1, 2, 3])
    check(ix.batch_search([[1], [3], [2, 1]], 0), orc.search(query_csr([[1], [3], [2, 1]]), 0))
    ix.close()


def test_failed_append_across_tiles_changes_nothing():
    """an append that rebuilds the last partial tile, builds a new one and then fails on a row of that new tile (a repeated
    hash) leaves rows, tiles, N, df and idf as they were, and a valid append continues from there"""
    corpus = multi_tile(12, 60_000)
    first, rest = slice_csr(corpus, 0, 20_000), slice_csr(corpus, 20_000, 60_000)
    bad = concat_csr([rest, cdb.sparse_csr([[(7, 1.0), (9, 0.5), (7, 2.0)]])])   # row 60000: in tile 1, not tile 0
    ix, orc = both(capacity_rows=70_000, capacity_pairs=len(bad[1]) + len(first[1]))
    ix.append(first, 1)
    orc.append(first, 1)
    qs = zipf_queries(13, 256, vocab=5000)
    hashes = np.concatenate([np.unique(corpus[1])[:1000], np.array([7, 9], np.uint32)])
    with pytest.raises(cdb.CosdataError) as e:
        ix.append(bad, 1)
    assert e.value.status == cdb.Status.INVALID_PARAMS
    assert len(ix) == 20_000
    check_stats(ix, orc, hashes)
    for k in (10, 0):
        check(ix.batch_search(qs, k), orc.search(query_csr(qs), k))
    ix.append(rest, 2)
    orc.append(rest, 2)
    assert len(ix) == 60_000
    check_stats(ix, orc, hashes)
    for k in (10, 0):
        check(ix.batch_search(qs, k), orc.search(query_csr(qs), k))
    ix.close()


def test_one_million_documents_batch_1024():
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < 8 << 30:
        pytest.skip("needs 8 GB of free device memory")
    n = 1_000_000
    chunks = [zipf_docs(100 + i, 250_000) for i in range(4)]
    corpus = concat_csr(chunks)
    ix, orc = both(capacity_rows=n, capacity_pairs=len(corpus[1]))
    for c in chunks:
        ix.append(c, 1)
    orc.append(corpus, 1)
    qs = zipf_queries(11, 1024)
    ids, scores, counts = ix.batch_search(qs, 10)
    sample = list(range(0, 1024, 64))
    want = orc.search(query_csr([qs[i] for i in sample]), 10)
    check((ids[sample], scores[sample], counts[sample]), want)
    ix.close()
