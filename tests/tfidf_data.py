"""Seeded inputs for the TF-IDF tests and tools/bench_tfidf.py: small adversarial corpora driven through appends and deletes
across versions, and Zipf corpora of (term_hash, tf) rows with tf from bm25_term_frequency."""
import numpy as np

from tests.sparse_data import zipf_csr

SPECIAL_TF = np.array([0.0, -0.0, -1.5, np.inf, -np.inf, np.nan, 1e-30, 3.0, 0.5], np.float32)


def random_rows(rng, n, vocab, max_terms=6, special=0.15, uncounted=0.1):
    """-> (rows [[(hash, tf)]], counted u8[n]); hashes of a row distinct, uncounted rows empty"""
    rows, counted = [], np.ones(n, np.uint8)
    for r in range(n):
        if rng.random() < uncounted:
            rows.append([])
            counted[r] = 0
            continue
        m = int(rng.integers(0, min(max_terms, len(vocab)) + 1))
        hs = rng.choice(vocab, m, replace=False)
        tf = (rng.random(m) * 2.0).astype(np.float32)
        pick = rng.random(m) < special
        tf[pick] = SPECIAL_TF[rng.integers(0, len(SPECIAL_TF), int(pick.sum()))]
        rows.append(list(zip(hs.tolist(), tf.tolist())))
    return rows, counted


def op_script(seed, steps=6, vocab_size=10, rows_per_step=30, special=0.15):
    """a sequence of ('append', rows, counted, version) / ('delete', rows, version) with non-decreasing versions; deletes hit
    rows of the current and of older versions, and sometimes rows deleted before"""
    rng = np.random.default_rng(seed)
    vocab = rng.choice(1 << 31, vocab_size, replace=False).astype(np.uint32)
    ops, n, version = [], 0, int(rng.integers(1, 5))
    for _ in range(steps):
        version += int(rng.integers(0, 2))
        m = int(rng.integers(0, rows_per_step + 1))
        rows, counted = random_rows(rng, m, vocab, special=special)
        ops.append(("append", rows, counted, version))
        n += m
        if n and rng.random() < 0.8:
            if rng.random() < 0.5:
                version += 1
            dels = rng.choice(n, int(rng.integers(1, max(2, n // 4))), replace=True).astype(np.uint32)
            ops.append(("delete", dels, version))
    return vocab, ops


def random_queries(rng, vocab, nq, max_terms=8, absent=0.1):
    """hash lists with repeats and hashes absent from the index"""
    qs = []
    for _ in range(nq):
        m = int(rng.integers(0, max_terms + 1))
        q = rng.choice(vocab, m).tolist()
        q = [int(rng.integers(1 << 31, 1 << 32)) if rng.random() < absent else h for h in q]
        qs.append(q)
    return qs


def query_csr(qs):
    off = np.zeros(len(qs) + 1, np.uint64)
    if qs:
        off[1:] = np.cumsum([len(q) for q in qs])
    return off, np.array([h for q in qs for h in q], np.uint32)


def zipf_docs(seed, n_rows, vocab=1_000_000, mean_terms=40, avgdl=60.0, k1=1.2, b=0.75):
    """(offsets, hashes, tf) with Zipf term popularity (shared across seeds), tf = bm25_term_frequency of a small count over
    a document length drawn around avgdl"""
    from cosdata_b200 import bm25_term_frequency
    off, dims, _ = zipf_csr(seed, n_rows, vocab=vocab, mean_pairs=mean_terms)
    # zipf_csr's re-draw of a repeated dim can land on another dim of the row: drop such repeats (an index rejects them)
    row = np.repeat(np.arange(n_rows), np.diff(off).astype(np.int64))
    order = np.lexsort((dims, row))
    rep = np.zeros(dims.size, bool)
    rep[order[1:]] = (dims[order[1:]] == dims[order[:-1]]) & (row[order[1:]] == row[order[:-1]])
    dims = dims[~rep]
    off = np.zeros(n_rows + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(row[~rep], minlength=n_rows))
    rng = np.random.default_rng(seed + 7919)
    lens = np.diff(off).astype(np.int64)
    doc_len = np.repeat(lens + rng.poisson(avgdl - mean_terms, n_rows), lens).astype(np.uint32)
    count = rng.geometric(0.6, dims.size).astype(np.uint32)
    tf = bm25_term_frequency(count, doc_len, avgdl, k1, b)
    hashes = (dims.astype(np.uint64) * 2654435761 % (1 << 32)).astype(np.uint32)   # a bijection of the dims
    return off, hashes, tf


def zipf_queries(seed, nq, vocab=1_000_000, lo=3, hi=12):
    """query hash lists of lo..hi terms under the corpus' popularity"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(lo, hi + 1, nq)
    off, dims, _ = zipf_csr(seed + 1, nq, vocab=vocab, mean_pairs=hi + 8)
    qs = []
    for i in range(nq):
        d = dims[int(off[i]):int(off[i + 1])][:int(lens[i])]
        qs.append((d.astype(np.uint64) * 2654435761 % (1 << 32)).astype(np.uint32).tolist())
    return qs
