"""fp16 emulation of the tensor-core prefilter and an adversarial corpus for its error bound (CPU only).

The prefilter (csrc/tensor_scan.cu, f16 form) scores a query against a row as
    a = sum_i qh_i * xh_i,   xh = fp16_rne(f32(x) / |x|),   |x| = sqrt of the sequential f32 fold of x_i*x_i
and keeps a row only if a >= A_k - 2*eps(D), where A_k is the k-th largest of NG class maxima (class = row mod NG).
Products of two halfs are exact in f64, so `approx_scores` reproduces a up to the order of the f32 tensor accumulation.

The adversarial construction works on the normalised vectors: it puts every entry just above or just below an fp16
rounding midpoint, so that every entry rounds the same way by ~u = 2^-11 relative, and then adds one "ballast" entry on
a coordinate of its own that brings the norm to 1 (f32 normalisation then moves nothing across a midpoint):
  * entries are 2^-e * (1 + 2^-11 + off): off = +2^-23 rounds up, off = -2^-16 (query) / -2^-17 (targets) rounds down;
  * a row holds 3 entries at each of 2^-1 .. 2^-5 (sum of squares ~ 1 - 2^-10); each half of the query holds
    1 x 2^-1, 3 each at 2^-2 .. 2^-5 and 2 x 2^-6 (half of that);
  * the query rounds up on coordinate group G1 and down on G2;
  * decoys live on G1 and round up (approximate score too high), targets live on G2 and round down (too low).
Decoys and targets pair their levels with the query's identically, so their exact cosines agree to ~1e-6; the targets
share the query's ballast coordinate, which lifts every target's exact cosine just above every decoy's.  The approximate
scores then differ by ~1.29e-3 in the decoys' favour: more than eps(D) for D <= 128, so a filter at A_k - eps would
lose the targets (the true top-k), while A_k - 2*eps keeps them.
"""
import os
import re

import numpy as np

import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32

QL = np.array([1] + [2] * 3 + [3] * 3 + [4] * 3 + [5] * 3 + [6] * 2)   # one half of the query: sum 4^-e = (1 - 2^-10) / 2
RL = np.array([1] * 3 + [2] * 3 + [3] * 3 + [4] * 3 + [5] * 3)          # a row: sum 4^-e = 1 - 2^-10
UP, Q_DOWN, T_DOWN = 2.0 ** -23, -2.0 ** -16, -2.0 ** -17
BLOCK = 128                 # rows of one adversarial block: 64 targets, then 64 decoys (64 consecutive residues)
NT = ND = 64


def eps_coefficients():
    """(c0, c1) of prefilter_eps(dim) = c0 + c1 * dim, read from csrc/api.cu so the tests follow the bound."""
    with open(os.path.join(ROOT, "cosdata_b200", "csrc", "api.cu")) as f:
        src = f.read()
    m = re.search(r"prefilter_eps\(uint32_t dim\)\s*\{\s*return\s*([0-9.eE+-]+)f\s*\+\s*([0-9.eE+-]+)f\s*\*\s*\(float\)dim;", src)
    assert m, "prefilter_eps not found in csrc/api.cu"
    return float(m.group(1)), float(m.group(2))


def eps(dim):
    c0, c1 = eps_coefficients()
    return float(F32(c0) + F32(F32(c1) * F32(dim)))


def ng_for_k(k):
    """number of row classes the f16 form uses for a given k (launch_tensor_scan in csrc/tensor_scan.cu)"""
    return 16 if k <= 12 else (32 if k <= 28 else 64)


def seq_norm(m):
    """|x| of every row: sqrt of the sequential f32 fold of f32(x*x) (vector_store.rs:412), as the kernels compute it"""
    m = np.ascontiguousarray(m, dtype=F32)
    s = np.zeros(m.shape[0], F32)
    for c in range(m.shape[1]):
        s = (s + m[:, c] * m[:, c]).astype(F32)
    return np.sqrt(s).astype(F32)


def shadow(m):
    """fp16 copy of x / |x| (normalize_f16_kernel / prep_queries_kernel); degenerate norms give a zero row"""
    m = np.ascontiguousarray(m, dtype=F32)
    n = seq_norm(m)
    ok = (n >= F32(1e-15)) & (n <= F32(1e15))
    out = (m / np.where(ok, n, F32(1))[:, None]).astype(np.float16)
    out[~ok] = 0
    return out


def approx_scores(queries, rows):
    """a[q, r]: exact f64 sum of the products of the fp16 shadows"""
    return shadow(queries).astype(np.float64) @ shadow(rows).astype(np.float64).T


def cos_ref(query, rows):
    """reference cosine (oracle DistanceMetric::calculate on f32 storage) of one query against each row"""
    q = np.ascontiguousarray(query, dtype=F32)
    qm = orc.mag_f32(q)
    out = np.empty(len(rows))
    for i, r in enumerate(np.ascontiguousarray(rows, dtype=F32)):
        rc, v = orc.distance(0, 5, q.size, q.view(np.uint8), qm, r.view(np.uint8), orc.mag_f32(r))
        assert rc == 0
        out[i] = v
    return out


def _level_values(levels, off):
    return 2.0 ** -levels.astype(np.float64) * (1.0 + 2.0 ** -11 + off)


def _ballast(v, c):
    r = 1.0 - (v * v).sum()
    assert r >= 0
    v[c] = np.sqrt(r)


def _arrangements():
    """row level for each of the 15 query coordinates of a half (query levels QL, sorted pairing), 81 distinct ways:
    the three coordinates of each query level 2..5 receive the row levels {e-1, e-1, e} in any of three orders, which
    leaves the dot product with the query unchanged"""
    base = np.sort(RL)
    out = []
    for code in range(81):
        lv = base.copy()
        for j, start in enumerate((1, 4, 7, 10)):
            tri = np.array([base[start], base[start], base[start + 2]])
            lv[start:start + 3] = np.roll(tri, (code // 3 ** j) % 3)
        out.append(lv)
    return out


def block(dim, seed):
    """One adversarial block -> (query [dim], targets [64, dim], decoys [64, dim]), all f32.  The 32 coordinates it uses
    (G1, G2, the query/target ballast, the decoy ballast) and the signs are drawn from `seed`, so blocks of different seeds
    are far apart from each other."""
    assert dim >= 32
    rng = np.random.default_rng(seed)
    coords = rng.permutation(dim)
    g1, g2, bqt, bd = coords[:15], coords[15:30], coords[30], coords[31]
    sign = np.where(rng.random(dim) < 0.5, -1.0, 1.0)
    q = np.zeros(dim)
    q[g1], q[g2] = _level_values(QL, UP), _level_values(QL, Q_DOWN)
    _ballast(q, bqt)
    arr = _arrangements()
    pick = rng.permutation(len(arr))
    targets, decoys = np.zeros((NT, dim)), np.zeros((ND, dim))
    for i in range(NT):
        targets[i, g2] = _level_values(arr[pick[i]], T_DOWN)
        _ballast(targets[i], bqt)
    for i in range(ND):
        decoys[i, g1] = _level_values(arr[pick[i]], UP)
        _ballast(decoys[i], bd)
    f = lambda m: (m * sign).astype(F32)
    return f(q), f(targets), f(decoys), (g1, g2)


def same_vector(dim, seed):
    """a row that rounds up on every entry, used as its own query: cosine ~1, both sides round up (the tightest
    single-sided case)"""
    rng = np.random.default_rng(seed)
    coords = rng.permutation(dim)
    v = np.zeros(dim)
    v[coords[:15]] = _level_values(RL, UP)
    _ballast(v, coords[15])
    return (v * np.where(rng.random(dim) < 0.5, -1.0, 1.0)).astype(F32), coords[:15]


def rounding_signs(v, coords):
    """sign of (fp16 shadow - exact normalised value) at `coords` of each row, relative to the sign of the entry"""
    v = np.atleast_2d(np.ascontiguousarray(v, dtype=F32))
    exact = v.astype(np.float64) / seq_norm(v).astype(np.float64)[:, None]
    d = (shadow(v).astype(np.float64) - exact) * np.sign(exact)
    return np.sign(d[:, coords])


def noise(n, dim, queries, seed, max_cos=0.3):
    """n Gaussian rows whose cosine with every query is below max_cos"""
    rng = np.random.default_rng(seed)
    qn = queries.astype(np.float64) / np.linalg.norm(queries.astype(np.float64), axis=1)[:, None]
    out = np.empty((0, dim), F32)
    while len(out) < n:
        x = rng.standard_normal((2 * n + 64, dim)).astype(F32)
        c = (x.astype(np.float64) @ qn.T) / np.linalg.norm(x.astype(np.float64), axis=1)[:, None]
        out = np.concatenate([out, x[(c < max_cos).all(axis=1)]])
    return out[:n]


def corpus(n, dim, nq, seed):
    """Adversarial corpus -> (rows [n, dim], queries [nq, dim], blocks).  Query j uses block j % blocks, whose rows are
    [b*128, b*128+64) targets and [b*128+64, b*128+128) decoys; the rest is low-cosine noise.  Every block lies inside the
    first 16384 rows, the prefix the prefilter's seeding pass reads."""
    nb = max(1, min(nq, 16, (n - 1024) // BLOCK))
    qs, rows = [], []
    for b in range(nb):
        q, t, d, _ = block(dim, seed * 1000 + b)
        qs.append(q)
        rows += [t, d]
    base = np.stack(qs)
    x = np.concatenate(rows + [noise(n - nb * BLOCK, dim, base, seed)])
    return x, base[np.arange(nq) % nb], nb


def filter_keeps(a_row, k, margin):
    """rows of one query the f16 filter keeps: a >= (k-th largest class maximum) - margin, class = row mod NG"""
    ng = ng_for_k(k)
    n = a_row.size
    pad = np.full((-n) % ng, -np.inf)
    cmax = np.concatenate([a_row, pad]).reshape(-1, ng).max(axis=0)
    a_k = np.sort(cmax)[::-1][k - 1]
    return a_row >= a_k - margin
