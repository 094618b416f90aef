"""numpy emulation of the s8 form of the prefilter (csrc/tensor_scan.cu, KIND 2; DESIGN.md section 5c) and an adversarial
corpus for its error bound (CPU only).

Quantization, per corpus tile T of 256 rows aligned to row 0 and per query:
    x_hat = f32(x / |x|)  (|x| = sequential f32 norm; degenerate norms give a zero row that has no say in s_T / E_T)
    s_T = f32(max over the tile's proper rows of max_i |x_hat_i| / 127),  c = rint(f32(x_hat / s_T)) in [-127, 127]
    E_T >= max over the tile's proper rows of |x_hat - s_T c|  (f64, rounded up to f32);  likewise s_q, c_q, e_q per query
The approximate score is a = s_T s_q (c_q . c_x) and the bound
    eps(q, T) = (1 + delta_n + e_q) E_T + e_q (1 + delta_n) + delta_ref(D)
follows from q_hat . x_hat = s_q s_T (c_q . c_x) + s_q c_q . r_x + r_q . x_hat with Cauchy-Schwarz on the two residual terms.

The adversarial block puts every entry of its rows just beside an s8 rounding midpoint of the tile's scale, with the
residuals aligned with the query (targets: rounded down, the approximate score too low by ~E_T) or against it (decoys:
rounded up, too high by ~E_T).  The targets also share a ballast coordinate with the query, which lifts their exact cosine
just above the decoys'.  The decoys' approximate scores then lead the targets' by more than eps: a filter at eps/2 loses the
true top-k, the filter at eps keeps it.
"""
import os
import re

import numpy as np

from tests import prefilter_adversary as pa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
TILE = 256
U = 2.0 ** -24


def delta_coefficients():
    """(n0, r1, r0): delta_n = (D + n0) u and delta_ref = (r1 D + r0) u, read from csrc/tensor_scan.cu"""
    with open(os.path.join(ROOT, "cosdata_b200", "csrc", "tensor_scan.cu")) as f:
        src = f.read()
    mn = re.search(r"a\.dn1 = f32_up\(1\.0 \+ \(\(double\)dim \+ ([0-9.]+)\) \* 0x1p-24\);", src)
    mr = re.search(r"a\.dref = f32_up\(\(([0-9.]+) \* dim \+ ([0-9.]+)\) \* 0x1p-24\);", src)
    assert mn and mr, "dn1 / dref not found in csrc/tensor_scan.cu"
    return float(mn.group(1)), float(mr.group(1)), float(mr.group(2))


def deltas(dim):
    n0, r1, r0 = delta_coefficients()
    return (dim + n0) * U, (r1 * dim + r0) * U


def _up(x):
    """smallest f32 >= x (x >= 0, f64)"""
    f = np.float32(x)
    return float(np.nextafter(f, F32(np.inf))) if float(f) < x else float(f)


def normalized(m):
    """x_hat rows (f32) and the proper-row mask, as normalize_f16_kernel / prep_queries_kernel compute them"""
    m = np.ascontiguousarray(m, dtype=F32)
    n = pa.seq_norm(m)
    ok = (n >= F32(1e-15)) & (n <= F32(1e15))
    xh = (m / np.where(ok, n, F32(1))[:, None]).astype(F32)
    xh[~ok] = 0
    return xh, ok


def quantize_set(xh, ok):
    """one scale for the rows of xh (a corpus tile, or a single query) -> (codes int64, s f32, E f32)"""
    mx = F32(np.abs(xh[ok]).max()) if ok.any() else F32(0)
    s = F32(mx / F32(127)) if mx > 0 else F32(0)
    if s > 0:
        c = np.clip(np.rint((xh / s).astype(F32)), -127, 127).astype(np.int64)
    else:
        c = np.zeros(xh.shape, np.int64)
    c[~ok] = 0
    r = xh.astype(np.float64) - np.float64(s) * c
    e = np.sqrt((r[ok] ** 2).sum(axis=1)).max() if ok.any() else 0.0
    return c, s, _up(e * (1 + 2.0 ** -30))


def quantize_corpus(x, deleted=None):
    """-> (codes [n, D], s_T [tiles], E_T [tiles]) with tiles of 256 rows aligned to row 0.  deleted (bool [n], may be
    None): those rows get zero codes and no say in s_T / E_T, as in quantize_s8_tiles_kernel"""
    xh, ok = normalized(x)
    if deleted is not None:
        ok = ok & ~np.asarray(deleted, bool)
    codes = np.zeros(xh.shape, np.int64)
    nt = (len(x) + TILE - 1) // TILE
    s, e = np.zeros(nt, F32), np.zeros(nt)
    for t in range(nt):
        sl = slice(t * TILE, (t + 1) * TILE)
        codes[sl], s[t], e[t] = quantize_set(xh[sl], ok[sl])
    return codes, s, e


def quantize_queries(q):
    xh, ok = normalized(q)
    out = [quantize_set(xh[i:i + 1], ok[i:i + 1]) for i in range(len(q))]
    return np.concatenate([o[0] for o in out]), np.array([o[1] for o in out], F32), np.array([o[2] for o in out])


def filter_terms(queries, rows, deleted=None, corpus=None):
    """-> (dp, s, eps), each [nq, n] f64: the exact s32 dot product c_q . c_x of the codes, s = s_T s_q and eps(q, T(r)).
    The float64 product of the integer codes is exact: |dp| <= 127^2 D < 2^53.  corpus: quantize_corpus(rows, deleted)
    if the caller has it already."""
    dim = rows.shape[1]
    cx, sx, ex = corpus if corpus is not None else quantize_corpus(rows, deleted)
    cq, sq, eq = quantize_queries(queries)
    tile = np.arange(len(rows)) // TILE
    dp = cq.astype(np.float64) @ cx.astype(np.float64).T
    s = sq.astype(np.float64)[:, None] * sx.astype(np.float64)[tile][None, :]
    dn, dref = deltas(dim)
    e = (1 + dn + eq[:, None]) * ex[tile][None, :] + eq[:, None] * (1 + dn) + dref
    return dp, s, e


def scores_and_eps(queries, rows, deleted=None):
    """a[q, r] = s_T s_q (c_q . c_x) (f64) and eps[q, r] = eps(q, T(r))"""
    dp, s, e = filter_terms(queries, rows, deleted)
    return dp * s, e


def class_maxima(lb, ng, use=None):
    """-> (maxima [nq, ng], argmax rows [nq, ng]) of lb [nq, n] over the classes row mod ng; rows where use [nq, n] (or
    [n]) is False have no say, an empty class is -inf"""
    nq, n = lb.shape
    v = np.where(use, lb, -np.inf) if use is not None else lb
    v = np.concatenate([v, np.full((nq, (-n) % ng), -np.inf)], axis=1).reshape(nq, -1, ng)
    j = v.argmax(axis=1)
    return np.take_along_axis(v, j[:, None, :], axis=1)[:, 0, :], j * ng + np.arange(ng)[None, :]


def kth_largest(cm, k):
    """A = the k-th largest of each query's class maxima"""
    return np.sort(cm, axis=1)[:, cm.shape[1] - k]


def filter_bounds(dp, s, e, k, has_deg, seed_rows):
    """-> (A*, A_seed) per query: the k-th largest class maximum of the lower bounds a - eps over all rows, and over the
    seeding pass's row prefix [0, seed_rows).  has_deg: rows with dp == 0 have no say (the HAS_DEG rule: a deleted or
    degenerate row has a zero code row, and the kernel cannot tell it from a proper row that scores exactly 0)."""
    ng = pa.ng_for_k(k)
    lb = dp * s - e
    use = dp != 0 if has_deg else np.ones(dp.shape, bool)
    a_all = kth_largest(class_maxima(lb, ng, use)[0], k)
    m = min(seed_rows, dp.shape[1])
    a_seed = kth_largest(class_maxima(lb[:, :m], ng, use[:, :m])[0], k)
    return a_all, a_seed


def filter_keeps(a_row, e_row, k, scale=1.0):
    """rows of one query the s8 filter keeps: class maxima of the lower bounds a - eps (class = row mod NG), A = their
    k-th largest, keep a + eps >= A.  scale < 1 weakens eps on both sides."""
    ng = pa.ng_for_k(k)
    lo = a_row - scale * e_row
    pad = np.full((-lo.size) % ng, -np.inf)
    cmax = np.concatenate([lo, pad]).reshape(-1, ng).max(axis=0)
    A = np.sort(cmax)[::-1][k - 1]
    return a_row + scale * e_row >= A


def adversarial_block(dim, seed, nt=64, nd=64):
    """-> (query [dim], rows [1 + nt + nd, dim]): a spike row that fixes the tile's scale at f32(1/127), nt targets, nd
    decoys.  Fits one corpus tile when placed at a multiple of 256."""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(dim)
    spike, bq, bd, main = perm[0], perm[1], perm[2], perm[3:]
    m = len(main)
    sign = np.where(rng.random(dim) < 0.5, -1.0, 1.0)
    s_t = float(F32(1.0) / F32(127))
    lvl = np.floor(0.9 * 127 / np.sqrt(m) - 0.5)                 # main entries sit at (lvl + 1/2 -+ d) s_T
    gamma_t = np.sqrt(1 - ((lvl + 0.5) * s_t) ** 2 * m)          # target ballast (on the query's ballast coordinate)
    beta = min(1.0, 0.25 * m * s_t / gamma_t)                    # query ballast: lifts targets by ~ E_T / 2
    q = np.zeros(dim)
    q[main], q[bq] = 1.0, beta
    rows = np.zeros((1 + nt + nd, dim))
    rows[0, spike] = 1.0
    for i in range(nt):
        d = 0.01 + 0.0005 * i
        rows[1 + i, main] = (lvl + 0.5 - d) * s_t
        rows[1 + i, bq] = np.sqrt(1 - (rows[1 + i, main] ** 2).sum())
    for i in range(nd):
        d = 0.01 + 0.0005 * i
        rows[1 + nt + i, main] = (lvl + 0.5 + d) * s_t
        rows[1 + nt + i, bd] = np.sqrt(1 - (rows[1 + nt + i, main] ** 2).sum())
    return (q * sign).astype(F32), (rows * sign).astype(F32)


def adversarial_corpus(n, dim, nq, seed):
    """-> (rows [n, dim], queries [nq, dim], blocks): block b occupies tile b (rows [256 b, 256 b + 129)), the rest of the
    corpus is low-cosine noise; query j uses block j % blocks.  Every block lies in the first 16384 rows."""
    nb = max(1, min(nq, 16, n // TILE - 1))
    x = pa.noise(n, dim, np.ones((1, dim), F32), seed, max_cos=0.3)
    qs = []
    for b in range(nb):
        q, r = adversarial_block(dim, seed * 1000 + b)
        x[b * TILE:b * TILE + len(r)] = r
        qs.append(q)
    base = np.stack(qs)
    return x, base[np.arange(nq) % nb], nb
