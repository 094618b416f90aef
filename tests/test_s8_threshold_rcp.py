"""The integer threshold of the s8 prefilter (csrc/tensor_scan.cu, tensor_scan_s8_kernel; DESIGN.md section 5c) without a
division, emulated with exact rational arithmetic and directed rounding.

A row is emitted iff its s32 dot product dp >= thrI, so thrI must not exceed (A - eps) / (s_T * s_q); a lower thrI only
adds candidates, which the exact re-rank removes again.  Both forms are such lower bounds, and neither is always the
lower of the two (each rounds twice), so the tests check the reciprocal form against the exact quotient, and against
the division form: within 1 while |thrI| < 2^21 (each form is within 4 roundings of the quotient, a relative 2^-21
beyond that), and where the division gives NaN -> 0 or +-inf, the same result or a lower one.

The division form (tensor_scan_kernel, KIND 2) computes
    thrI = floor(fl_down(num / s)),  s = fl_up(s_T * s_q) for num >= 0, fl_down(s_T * s_q) otherwise,
the reciprocal form (tensor_scan_s8_kernel)
    thrI = floor(fl_down(fl_down(num * r_T) * r_q)),  r = fl_down(1 / s) for num >= 0, fl_up(1 / s) otherwise,
with num = fl_down(A - eps) and the reciprocals of quantize_s8_tiles_kernel / prep_queries_kernel.  The float -> int
conversion is cvt.rmi.s32.f32: NaN -> 0, saturating at INT_MIN / INT_MAX.
"""
from fractions import Fraction
import math

import numpy as np
import pytest

F32 = np.float32
MAXF = Fraction(float(np.finfo(F32).max))
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


def _round(x, up):
    """x (exact rational) rounded to f32 downward / upward, overflow as IEEE directed rounding does"""
    if x > MAXF:
        return F32(np.inf) if up else F32(MAXF)
    if x < -MAXF:
        return F32(-MAXF) if up else F32(-np.inf)
    f = F32(float(x))
    while Fraction(float(f)) > x and not up:
        f = np.nextafter(f, F32(-np.inf))
    while Fraction(float(f)) < x and up:
        f = np.nextafter(f, F32(np.inf))
    return f


def _mul(a, b, up):
    a, b = float(a), float(b)
    if math.isnan(a) or math.isnan(b):
        return F32(np.nan)
    if math.isinf(a) or math.isinf(b):
        if a == 0.0 or b == 0.0:
            return F32(np.nan)
        return F32(math.copysign(np.inf, a) * math.copysign(1.0, b))
    return _round(Fraction(a) * Fraction(b), up)


def _div(a, b, up):
    a, b = float(a), float(b)
    if math.isnan(a) or math.isnan(b) or (a == 0.0 and b == 0.0) or (math.isinf(a) and math.isinf(b)):
        return F32(np.nan)
    if b == 0.0 or math.isinf(a):
        return F32(math.copysign(np.inf, a) * math.copysign(1.0, b))
    if math.isinf(b):
        return F32(0.0)
    return _round(Fraction(a) / Fraction(b), up)


def _rcp(s, up):
    return _div(F32(1.0), s, up)


def _f2i_rd(x):
    x = float(x)
    if math.isnan(x):
        return 0
    if x >= 2.0 ** 31:
        return INT_MAX
    if x < -(2.0 ** 31):
        return INT_MIN
    return math.floor(x)


def thr_division(num, st, sq):
    s = _mul(st, sq, True) if num >= 0 else _mul(st, sq, False)
    return _f2i_rd(_div(num, s, False))


def thr_reciprocal(num, st, sq):
    up = not num >= 0
    return _f2i_rd(_mul(_mul(num, _rcp(st, up), False), _rcp(sq, up), False))


def _exact_floor(num, st, sq):
    """floor((A - eps) / (s_T s_q)) for finite num and positive scales, saturated like the conversion"""
    q = Fraction(float(num)) / (Fraction(float(st)) * Fraction(float(sq)))
    return max(INT_MIN, min(INT_MAX, math.floor(q)))


def _check(num, st, sq, within_one=True):
    num, st, sq = F32(num), F32(st), F32(sq)
    old, new = thr_division(num, st, sq), thr_reciprocal(num, st, sq)
    if math.isfinite(num) and st > 0 and sq > 0:
        exact = _exact_floor(num, st, sq)
        assert old <= exact and new <= exact, (num, st, sq, old, new, exact)
        if within_one:
            assert abs(old - new) <= 1 + abs(exact) * 2.0 ** -21, (num, st, sq, old, new)
    else:
        assert new <= old, (num, st, sq, old, new)
    return old, new


def test_random_scales():
    # the headline's scales: s = max |x_hat_i| / 127 of unit rows, bounds A - eps within [-1 - eps, 1]
    rng = np.random.default_rng(5)
    n_within_one = 0
    for _ in range(3000):
        st = F32(rng.uniform(0.02, 1.0) / 127)
        sq = F32(rng.uniform(0.02, 1.0) / 127)
        old, new = _check(F32(rng.uniform(-1.05, 1.0)), st, sq)
        n_within_one += abs(old - new) <= 1
    assert n_within_one >= 2990


def test_exact_reciprocals_and_wide_scales():
    rng = np.random.default_rng(6)
    # powers of two: the reciprocals are exact, both forms agree
    for e in range(-20, -2):
        for num in (F32(0.75), F32(-0.3), F32(1e-3)):
            old, new = _check(num, F32(2.0 ** e), F32(2.0 ** -8))
            assert old == new
    # scales over many binades; the quotient saturates the conversion at the large end
    for _ in range(2000):
        st = F32(10.0 ** rng.uniform(-12, 0))
        sq = F32(10.0 ** rng.uniform(-12, 0))
        num = F32(rng.uniform(-2, 2) * 10.0 ** rng.uniform(-6, 0))
        _check(num, st, sq)


def test_subnormal_and_extreme_scales():
    tiny = F32(np.finfo(F32).smallest_subnormal)
    cases = []
    for s in (tiny, F32(1e-40), F32(np.finfo(F32).tiny), F32(1e-30), F32(3e-39)):
        for other in (s, F32(1.0 / 127), F32(1e-3)):
            for num in (F32(0.5), F32(-0.5), F32(1e-30), F32(-1e-30), F32(1e-45), F32(-1e-45)):
                cases.append((num, s, other))
                cases.append((num, other, s))
    for num, st, sq in cases:
        # the reciprocal of a subnormal scale can overflow (rounded down: FLT_MAX), so only the bound itself holds in general
        old, new = _check(num, st, sq, within_one=False)
        if old in (INT_MIN, INT_MAX) and not (st < np.finfo(F32).tiny or sq < np.finfo(F32).tiny):
            assert new == old


@pytest.mark.parametrize("num", [F32(0.0), F32(-0.0)])
def test_zero_numerator(num):
    for st, sq in ((F32(0.004), F32(0.006)), (F32(0.0), F32(0.006)), (F32(0.004), F32(0.0)), (F32(0.0), F32(0.0))):
        old, new = _check(num, st, sq)
        assert old == new == 0


def test_minus_infinity_bound():
    # no bound yet: A = -inf, every row passes
    for st, sq in ((F32(0.004), F32(0.006)), (F32(0.0), F32(0.006)), (F32(0.004), F32(0.0)), (F32(0.0), F32(0.0))):
        old, new = _check(F32(-np.inf), st, sq)
        assert old == new == INT_MIN


def test_zero_scales():
    # s_T = 0: an all-degenerate or all-deleted tile (every code 0, dp = 0); s_q = 0: a zero or padding query.  The division
    # gives +-inf (saturated) or NaN -> 0; the reciprocal form must give the same or lower.
    for num in (F32(0.7), F32(-0.7), F32(1e-20), F32(-1e-20), F32(np.inf)):
        for st, sq in ((F32(0.0), F32(0.006)), (F32(0.004), F32(0.0)), (F32(0.0), F32(0.0))):
            old, new = _check(num, st, sq)
            assert old == new
            assert new == (INT_MAX if num > 0 else INT_MIN)
