"""The sparse oracle (tests/sparse_oracle.c) pinned by an independent pure-Python restatement of the reference text:
InvertedIndexNode::quantize (inverted_index.rs:168-172), SparseAnnQueryBasic::sequential_search (sparse_ann_query.rs:68-147)
with its hash-map accumulation and touched semantics, finalize_sparse_ann_results (inverted/mod.rs:331-381) and the
sampling decision (inverted/mod.rs:148-247).  CPU only."""
import math
import struct

import numpy as np
import pytest

from tests import pysparse as ps
from tests.sparse_data import big_sim_rows, quirky_rows

F = np.float32


def as_u(x, hi):
    """Rust `f32 as u8 / u32`: saturating, NaN -> 0"""
    x = float(x)
    if math.isnan(x) or x <= 0:
        return 0
    return hi if x >= hi else int(x)


def quantize(value, ub, bits):
    quantization = (1 << bits) - 1
    max_val = F(quantization)
    with np.errstate(all="ignore"):
        x = (F(value) / F(ub)) * max_val
    if not math.isnan(x):                       # f32::clamp(0.0, max_val); NaN stays NaN
        x = min(max(x, F(0)), max_val)
    return min(as_u(x, 255), quantization)


def thresholds(thr, bits):
    with np.errstate(all="ignore"):
        p = F(1 << bits) * F(thr)
    m = F(255) if math.isnan(p) else min(p, F(255))   # f32::min(NaN, 255) = 255
    return as_u(m, 255), as_u(F(thr) * F(1 << bits), 0xFFFFFFFF)


def total_key(v):
    b = struct.unpack("<I", struct.pack("<f", v))[0]
    if math.isnan(v):
        b = 0xFFC00000
    return (~b & 0xFFFFFFFF) if b & 0x80000000 else (b | 0x80000000)


def search(rows, query, k, bits, ub, thr, rerank, factor, id_base=0, deleted=()):
    one_quantized = (1 << bits) - 1
    etv, low = thresholds(thr, bits)
    lists = {}                                  # dim -> {key: [row, ...]}
    for r, pairs in enumerate(rows):
        for d, v in pairs:
            lists.setdefault(d, {}).setdefault(quantize(v, ub, bits), []).append(r)
    dot = {}
    for d, v in sorted(query, key=lambda p: -p[1] if not math.isnan(p[1]) else 0):
        node = lists.get(d)
        if node is None:
            continue
        qv = quantize(v, ub, bits)
        keys = range(one_quantized, -1, -1) if qv > low else range(one_quantized, etv - 1, -1)
        for key in keys:
            for r in node.get(key, []):
                if r in deleted:
                    continue
                dot[r] = (dot.get(r, 0) + qv * key) & 0xFFFFFFFF
    res = sorted(dot.items(), key=lambda x: (-x[1], x[0]))[: k * (factor if rerank else 1)]
    if not rerank:
        return [(r + id_base, F(s)) for r, s in res[:k]]
    out = []
    for r, _ in res:
        m = dict(rows[r])                       # the last pair of a dim wins
        dp = F(0)
        with np.errstate(all="ignore"):
            for d, qv in query:
                if d in m:
                    dp = F(dp + F(F(m[d]) * F(qv)))
        out.append((r + id_base, dp))
    out.sort(key=lambda x: (-total_key(x[1]), x[0]))
    return out[:k]


def compare(rows, queries, k, bits, ub, thr, rerank, factor=5, id_base=0, deleted=()):
    dl = None
    if deleted:
        dl = np.zeros(len(rows), np.uint8)
        dl[list(deleted)] = 1
    ids, scores, counts = ps.search(ps.csr(rows), ps.csr(queries), k, bits, ub, thr, rerank, factor, id_base, dl)
    for q, query in enumerate(queries):
        want = search(rows, query, k, bits, ub, thr, rerank, factor, id_base, set(deleted))
        assert counts[q] == len(want)
        assert ids[q, : len(want)].tolist() == [i for i, _ in want]
        got_bits = scores[q, : len(want)].view(np.uint32).tolist()
        want_bits = [0xFFC00000 if math.isnan(s) else int(np.array(s, F).view(np.uint32)) for _, s in want]
        assert got_bits == want_bits
        assert np.all(ids[q, len(want):] == 0xFFFFFFFF)


def test_quantize_and_thresholds():
    for bits in range(4, 9):
        for v in (0.0, -0.0, -1.0, 0.5, 0.999999, 1.0, 1.5, 1e30, float("nan"), float("inf"), 1e-40, 0.0666):
            for ub in (1.0, 3.0, 0.7):
                assert ps.quantize(v, ub, bits) == quantize(v, ub, bits), (v, ub, bits)
        for thr in (0.0, 0.5, 1.0, 1.7, -0.3, float("nan"), 1e12, float("inf")):
            assert ps.thresholds(thr, bits) == thresholds(thr, bits)
    assert thresholds(float("nan"), 4) == (255, 0)
    assert thresholds(1.0, 4) == (16, 16)


@pytest.mark.parametrize("bits", [4, 5, 6, 7, 8])
def test_search_matches_the_restatement(bits):
    rows = quirky_rows(bits, 300, 25)
    rows[0] = [(7, 0.0)]
    rows[1] = []
    rows[2] = [(3, 0.2), (3, 0.9), (3, 0.4)]
    queries = quirky_rows(50 + bits, 25, 30)
    queries[0] = []
    queries[1] = [(7, 0.0)]
    queries[2] = [(3, 0.5), (3, 0.5), (9, 2.0)]
    queries[3] = [(27, 1.0)]
    for thr in (0.0, 0.5, 1.0, 1.7, -0.3, float("nan")):
        for rerank, k in ((False, 5), (True, 4), (False, 1), (True, 400)):
            compare(rows, queries, k, bits, 1.5 if bits % 2 else 1.0, thr, rerank, id_base=9, deleted=(4, 5, 6) if bits == 5 else ())


def test_empty_key_range_and_ties():
    rows = [[(1, 0.1)], [(1, 0.9)], [(2, 0.5)]]
    ids, _, counts = ps.search(ps.csr(rows), ps.csr([[(1, 0.05)]]), 3, thr=1.0)
    assert counts[0] == 0
    rows = [[(0, 0.5)] for _ in range(20)]
    compare(rows, [[(0, 1.0)]], 5, 4, 1.0, 0.0, False)
    compare(rows, [[(0, 1.0)]], 3, 4, 1.0, 0.0, True, factor=2)


def test_sampling_decision():
    rng = np.random.default_rng(1)
    for vals in (rng.gamma(1.0, 1.5, 5000).astype(F), np.zeros(0, F), np.array([np.nan, 12.0, 1.0, 0.5], F)):
        for clamp in (1.0, 0.0, 50.0):
            counts, ub = ps.sample(vals, clamp)
            want = [int(np.sum(vals > F(t))) for t in range(1, 10)]
            assert counts.tolist() == want
            n = F(vals.size)
            with np.errstate(all="ignore"):
                pct = [(F(c) / n) * F(100) for c in want]
            w_ub = next((float(t + 1) for t, p in enumerate(pct) if p <= F(clamp)), 10.0)
            assert ub == w_ub
    assert ps.sample(np.zeros(0, F))[1] == 10.0


def test_similarities_above_2_24_and_wrapping():
    """selection and order on the u32 similarity (not its f32 image), u32 wrap-around, u32 -> f32 rounding of the score"""
    rows, query = big_sim_rows()
    qv = quantize(query[-1][1], 1.0, 8)
    raw = [len(r) - 1 and (len(r) - 1) * 100 * 255 * 255 + quantize(r[-1][1], 1.0, 8) * qv for r in rows]
    sims = sorted({x & 0xFFFFFFFF for x in raw})
    assert any(x >= 2 ** 32 for x in raw) and min(sims) >= 2 ** 24
    assert len({float(F(x)) for x in sims}) < len(sims)      # distinct u32 similarities that share an f32 image
    for k, rerank in ((1, False), (5, False), (20, False), (3, True)):
        compare(rows, [query], k, 8, 1.0, 0.0, rerank, factor=4)
