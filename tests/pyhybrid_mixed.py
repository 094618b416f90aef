"""Pure-Python restatement of batch_hybrid_search over a batch that mixes kinds (repo.rs:343-555): the query_mapping the
reference records while it sorts the queries into a dense, a sparse and a TF-IDF batch in request order, and the fusion
of each query from its two lists with tests/pyhybrid.fuse.  Test infrastructure only."""
import numpy as np

from tests.pyhybrid import fuse

KIND_SOURCES = (("dense", "sparse"), ("dense", "tfidf"), ("sparse", "tfidf"))   # CDB_HYBRID_* -> (first, second)


def query_mapping(kinds):
    """batch_hybrid_search's loop over the request: each query's (query_idx, idx1, idx2, kind), idx1 and idx2 its rows in
    the batches of the two sources its kind names, in request order -> (mapping, {source: batch size})"""
    n = {"dense": 0, "sparse": 0, "tfidf": 0}
    mapping = []
    for q, kind in enumerate(kinds):
        first, second = KIND_SOURCES[int(kind)]
        mapping.append((q, n[first], n[second], int(kind)))
        n[first] += 1
        n[second] += 1
    return mapping, n


def fuse_mixed(kinds, lists, k=60.0, dense_stride=1, ld_out=None):
    """the fusion of a mixed batch: lists = {source: (ids u32[n, ld], counts u32[n])}, each source's sub-search over its own
    batch (the queries whose kind names it, in request order); query q fuses row idx1 of its first source with row idx2
    of its second -> (ids u32[B, ld_out], scores f32[B, ld_out], counts u32[B]) in the library's output layout"""
    mapping, _ = query_mapping(kinds)
    ld_out = ld_out if ld_out is not None else max([0] + [lists[a][0].shape[1] + lists[b][0].shape[1]
                                                          for a, b in {KIND_SOURCES[int(x)] for x in kinds}])
    nq = len(mapping)
    ids = np.full((nq, ld_out), 0xFFFFFFFF, np.uint32)
    scores = np.zeros((nq, ld_out), np.float32)
    counts = np.zeros(nq, np.uint32)
    for q, i1, i2, kind in mapping:
        first, second = KIND_SOURCES[kind]
        (a, ca), (b, cb) = lists[first], lists[second]
        na, nb = min(int(ca[i1]), a.shape[1]), min(int(cb[i2]), b.shape[1])
        r = fuse(a[i1, :na].tolist(), b[i2, :nb].tolist(), k, "batch", (dense_stride if first == "dense" else 1, 1))
        counts[q] = len(r)
        for j, (key, s) in enumerate(r):
            ids[q, j] = key
            scores[q, j] = s
    return ids, scores, counts
