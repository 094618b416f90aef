"""Seeded sparse corpora for the sparse-index tests and tools/bench_sparse.py: SPLADE-like rows (Zipf-distributed dim
popularity, positive values) and adversarial ones (zero, negative and NaN values, duplicate dims)."""
import numpy as np


def zipf_csr(seed, n_rows, vocab=30522, mean_pairs=120, zipf_s=1.1, value_scale=1.0, dup=False, popularity_seed=0):
    """-> (offsets u64[n+1], dims u32, values f32).  Dims of a row are distinct unless dup.  Which dims are popular depends
    on popularity_seed and vocab only, so corpus pieces and queries drawn with different seeds share one vocabulary."""
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.poisson(mean_pairs, n_rows), 0, None).astype(np.int64)
    off = np.zeros(n_rows + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    total = int(off[-1])
    w = 1.0 / np.arange(1, vocab + 1) ** zipf_s
    cdf = np.cumsum(w / w.sum())
    perm = np.random.default_rng(popularity_seed).permutation(vocab).astype(np.uint32)
    dims = perm[np.minimum(np.searchsorted(cdf, rng.random(total)), vocab - 1)]
    if not dup and total:
        # make the dims of every row distinct: sort inside rows, bump repeats to unused neighbours
        row = np.repeat(np.arange(n_rows), lens)
        order = np.lexsort((dims, row))
        dims = dims[order]
        same = np.zeros(total, bool)
        same[1:] = (dims[1:] == dims[:-1]) & (row[1:] == row[:-1])
        dims[same] = (dims[same] + rng.integers(1, vocab, int(same.sum())).astype(np.uint32)) % vocab
        shuffle = np.argsort(row * 2.0 + rng.random(total), kind="stable")
        dims = dims[shuffle]
    vals = (rng.gamma(1.2, 0.6, total) * value_scale).astype(np.float32)
    return off, dims.astype(np.uint32), vals


def quirky_rows(seed, n_rows, vocab, max_len=12):
    """small rows over a small vocabulary with zero, negative, NaN, tiny and huge values and duplicate dims"""
    rng = np.random.default_rng(seed)
    specials = np.array([0.0, -0.5, np.nan, 1e-8, 3.0, 100.0, -0.0, 1.0, 0.999], np.float32)
    rows = []
    for _ in range(n_rows):
        m = int(rng.integers(0, max_len + 1))
        dims = rng.integers(0, vocab, m).astype(np.uint32)
        vals = rng.random(m).astype(np.float32) * np.float32(1.5)
        pick = rng.random(m) < 0.15
        vals[pick] = specials[rng.integers(0, len(specials), int(pick.sum()))]
        rows.append(list(zip(dims.tolist(), vals.tolist())))
    return rows


def big_sim_rows():
    """rows and a query whose u32 similarities (bits 8, values_upper_bound 1.0) lie above 2^24, where f32 no longer
    tells neighbours apart, and above 2^32, where they wrap: row = n x (0, 1.0) + (1, j/255) for j < 40, query = 100 x (0, 1.0) + (1, 2/255);
    each row's sim is n * 100 * 255 * 255 + key_j * qv (mod 2^32).  Every row appears twice (ties go to the smaller id)."""
    rows = []
    for n in (3, 700):
        for j in range(0, 40):
            r = [(0, 1.0)] * n + [(1, j / 255.0)]
            rows += [r, r]
    query = [(0, 1.0)] * 100 + [(1, 2 / 255.0)]
    return rows, query


def slice_csr(c, r0, r1):
    o, d, v = c
    a, b = int(o[r0]), int(o[r1])
    return (o[r0:r1 + 1] - o[r0]).astype(np.uint64), d[a:b], v[a:b]


def concat_csr(parts):
    offs, dims, vals, base = [np.zeros(1, np.uint64)], [], [], 0
    for o, d, v in parts:
        offs.append(o[1:] + np.uint64(base))
        dims.append(d)
        vals.append(v)
        base += int(o[-1])
    return np.concatenate(offs), np.concatenate(dims).astype(np.uint32), np.concatenate(vals).astype(np.float32)
