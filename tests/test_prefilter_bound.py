"""The fp16 prefilter's error bound eps(D) (prefilter_eps, csrc/api.cu) against an adversarial fp16 construction (CPU).

Soundness: |a - cos_ref| <= eps(D) for every pair the construction builds, including the tightest single-sided case.
Teeth: on the same corpus the filter at A_k - 2*eps keeps every true top-k row, and a filter at A_k - eps would lose
some, so the construction really comes within eps of the bound and a weaker margin would be caught.
"""
import numpy as np
import pytest

import oracle as orc
from tests import prefilter_adversary as pa

DIMS = [32, 33, 64, 100, 128, 256, 768, 1024, 4096]
KS = [1, 10, 12, 13, 28, 29, 64]


def test_eps_is_read_from_the_library_source():
    c0, c1 = pa.eps_coefficients()
    assert c0 > 0 and c1 > 0
    assert pa.eps(768) == pytest.approx(c0 + 768 * c1, rel=1e-6)


@pytest.mark.parametrize("dim", [32, 128, 768])
def test_construction_rounds_as_designed(dim):
    q, t, d, (g1, g2) = pa.block(dim, 11)
    assert (pa.rounding_signs(q, g1) > 0).all() and (pa.rounding_signs(q, g2) < 0).all()
    assert (pa.rounding_signs(d, g1) > 0).all(), "decoys must round up on every entry"
    assert (pa.rounding_signs(t, g2) < 0).all(), "targets must round down on every entry"
    assert len({r.tobytes() for r in np.concatenate([t, d])}) == pa.NT + pa.ND, "rows must be distinct"
    ct, cd = pa.cos_ref(q, t), pa.cos_ref(q, d)
    assert ct.min() >= cd.max(), "every target must be at least as close to the query as every decoy"
    a = pa.approx_scores(q[None], np.concatenate([t, d]))[0]
    assert a[pa.NT:].min() - a[:pa.NT].max() > 1.2e-3      # the fp16 errors push the decoys ahead of the targets
    v, c = pa.same_vector(dim, 12)
    assert (pa.rounding_signs(v, c) > 0).all()


@pytest.mark.parametrize("dim", DIMS)
def test_bound_is_sound_on_adversarial_pairs(dim):
    eps = pa.eps(dim)
    worst = 0.0
    for seed in range(3):
        q, t, d, _ = pa.block(dim, 100 * dim + seed)
        rows = np.concatenate([t, d, pa.noise(64, dim, q[None], seed)])
        err = pa.approx_scores(q[None], rows)[0] - pa.cos_ref(q, rows)
        assert np.abs(err).max() <= eps, (dim, np.abs(err).max(), eps)
        worst = max(worst, np.abs(err).max())
        v, _ = pa.same_vector(dim, 100 * dim + seed)
        e1 = pa.approx_scores(v[None], v[None])[0, 0] - pa.cos_ref(v, v[None])[0]
        assert 0 < e1 <= eps, (dim, e1, eps)
        worst = max(worst, e1)
    if dim <= 64:
        assert worst > 0.9 * eps      # the construction sits close to the bound where the bound is tightest


@pytest.mark.parametrize("dim", [d for d in DIMS if d <= 128])
def test_filter_margin_has_teeth(dim):
    n = 16 * pa.BLOCK + 2048
    x, qs, nb = pa.corpus(n, dim, 16, seed=dim)
    a = pa.approx_scores(qs, x)
    eps = pa.eps(dim)
    for k in KS:
        want_ids, _ = orc.brute_topk_f32(x, qs, k)
        for j in range(len(qs)):
            top = want_ids[j].astype(np.int64)
            b0 = (j % nb) * pa.BLOCK
            assert ((top >= b0) & (top < b0 + pa.NT)).all(), "the true top-k must be the block's targets"
            assert pa.filter_keeps(a[j], k, 2 * eps)[top].all(), (dim, k, j, "A_k - 2 eps lost a true top-k row")
            assert not pa.filter_keeps(a[j], k, eps)[top].all(), (dim, k, j, "A_k - eps keeps the whole top-k")
