"""Why the tensor-core prefilters must keep deleted rows out of the class maxima (DESIGN.md section 5): a CPU emulation of
the class-maximum filter.  A row survives iff its approximate score a >= A_k - 2*eps, A_k the k-th largest of the NG
class maxima.  When deleted rows (zero shadow rows score exactly 0, above every live row here) take part in the maxima,
the filter loses the live top-k; when they are left out, as the kernels do, it keeps it."""
import numpy as np
import pytest

NG, EPS = 16, 1e-3


def survivors(a, k, in_bound):
    """class-maximum filter over one query's approximate scores a; in_bound: rows allowed to set class maxima"""
    cls = np.arange(a.size) % NG
    cm = np.full(NG, -np.inf)
    np.maximum.at(cm, cls[in_bound], a[in_bound])
    thr = np.sort(cm)[::-1][k - 1] - 2 * EPS
    return np.flatnonzero(a >= thr)


@pytest.mark.parametrize("k", [1, 10])
def test_deleted_rows_in_the_bound_lose_the_live_top_k(k):
    rng = np.random.default_rng(1)
    n = 4096
    exact = -rng.uniform(0.6, 0.9, n)                          # all-negative live cosines
    deleted = np.zeros(n, bool)
    deleted[rng.choice(n, 3 * NG, replace=False)] = True     # deleted rows in every class
    deleted[np.arange(NG)] = True
    a = exact + rng.uniform(-EPS, EPS, n)                     # approximate scores within eps
    a[deleted] = 0.0                                          # zero shadow rows
    live = np.flatnonzero(~deleted)
    top = live[np.argsort(-exact[live], kind="stable")[:k]]
    kept_wrong = survivors(a, k, np.ones(n, bool))
    assert not np.isin(top, kept_wrong).any()                 # the bound over all rows drops every true top-k row
    kept = survivors(a, k, ~deleted)
    assert np.isin(top, kept).all()                           # the bound over live rows keeps them
