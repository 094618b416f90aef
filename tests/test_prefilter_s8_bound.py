"""The s8 prefilter's error bound eps(q, T) (DESIGN.md section 5c) against a numpy emulation of its quantization (CPU).

Soundness: |a - cos_ref| <= eps(q, T) for every pair, on uniform, clustered, outlier-dimension and adversarial data.
Teeth: on the adversarial corpus the filter at eps keeps every true top-k row, and a filter at eps/2 loses one.
"""
import numpy as np
import pytest

import oracle as orc
from tests import prefilter_adversary as pa
from tests import prefilter_s8 as ps

KS = [1, 10, 12, 13, 28, 29, 64]


def test_deltas_are_read_from_the_library_source():
    n0, r1, r0 = ps.delta_coefficients()
    assert n0 > 0 and r1 >= 1 and r0 > 0
    dn, dref = ps.deltas(768)
    assert 0 < dn < 1e-4 and 0 < dref < 1e-4


def _data(kind, n, dim, rng):
    if kind == "uniform":
        return rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    if kind == "clustered":
        c = rng.standard_normal((8, dim))
        return (c[rng.integers(0, 8, n)] + 0.05 * rng.standard_normal((n, dim))).astype(np.float32)
    if kind == "outliers":   # a few dimensions 30x larger than the rest: coarse scales, large residuals
        x = rng.standard_normal((n, dim))
        x[:, :4] *= 30
        return x.astype(np.float32)
    raise ValueError(kind)


def _check_sound(queries, rows):
    a, e = ps.scores_and_eps(queries, rows)
    worst = 0.0
    for j, q in enumerate(queries):
        err = np.abs(a[j] - pa.cos_ref(q, rows))
        assert (err <= e[j]).all(), (j, err.max(), e[j][err.argmax()])
        worst = max(worst, (err / e[j]).max())
    return worst


@pytest.mark.parametrize("kind", ["uniform", "clustered", "outliers"])
@pytest.mark.parametrize("dim", [32, 256, 768])
def test_bound_is_sound(kind, dim):
    rng = np.random.default_rng(dim + len(kind))
    rows = _data(kind, 600, dim, rng)                     # three tiles, the last one partial
    rows[5] = 0                                           # a degenerate row: zero codes, no say in s_T / E_T
    queries = np.concatenate([_data(kind, 3, dim, rng), rows[[7, 300]]])
    assert _check_sound(queries, np.delete(rows, 5, axis=0)) < 1.0


@pytest.mark.parametrize("dim", [64, 128, 256, 768])
def test_bound_is_sound_on_adversarial_pairs(dim):
    worst = 0.0
    for seed in range(2):
        q, rows = ps.adversarial_block(dim, 100 * dim + seed)
        worst = max(worst, _check_sound(q[None], rows))
    assert worst > 0.5          # the residuals line up with the query: the error reaches a good share of the bound


def test_degenerate_rows_do_not_set_the_scale():
    rng = np.random.default_rng(3)
    x = rng.uniform(-1, 1, (256, 64)).astype(np.float32)
    x[10] = 1e-30                     # norm underflows: degenerate
    codes, s, _ = ps.quantize_corpus(x)
    xh, ok = ps.normalized(x)
    assert not ok[10] and (codes[10] == 0).all()
    assert s[0] == np.float32(np.abs(xh[ok]).max() / np.float32(127))


@pytest.mark.parametrize("dim", [64, 128])
def test_filter_margin_has_teeth(dim):
    n = 16 * ps.TILE + 1024
    x, qs, nb = ps.adversarial_corpus(n, dim, 16, seed=dim)
    a, e = ps.scores_and_eps(qs, x)
    for k in KS:
        want_ids, _ = orc.brute_topk_f32(x, qs, k)
        for j in range(len(qs)):
            top = want_ids[j].astype(np.int64)
            b0 = (j % nb) * ps.TILE
            assert ((top > b0) & (top <= b0 + 64)).all(), "the true top-k must be the block's targets"
            assert ps.filter_keeps(a[j], e[j], k)[top].all(), (dim, k, j, "the filter at eps lost a true top-k row")
            assert not ps.filter_keeps(a[j], e[j], k, 0.5)[top].all(), (dim, k, j, "a filter at eps/2 keeps the top-k")
