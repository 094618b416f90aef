"""CPU checks of tests/pyhybrid.py, the restatement of the reference's reciprocal-rank fusion that the GPU tests compare
against: its f32 arithmetic against exact rational arithmetic rounded to nearest even, the two reference forms, the
association order of rank + k + EPSILON, NaN payloads, and the combining and no-truncation rules."""
import math
from fractions import Fraction

import numpy as np
import pytest

from tests import pyhybrid as ph

F32 = np.float32
MAX_F32 = Fraction(float(np.finfo(np.float32).max))


def rne_f32(x):
    """exact rational -> nearest f32, ties to even, subnormals included, overflow to inf"""
    if x == 0:
        return F32(0.0)
    sign, a = (-1 if x < 0 else 1), abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** max(e - 23, -149)
    m = a / q
    n = math.floor(m)
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    v = n * q
    if v > MAX_F32:
        return F32(sign * np.inf)
    return F32(sign * float(v))


def exact_contribution(rank, k):
    """1.0 / (rank + k + EPSILON) with each operation exact, then rounded once to f32; a +0 denominator gives +inf"""
    d1 = rne_f32(Fraction(rank) + Fraction(float(k)))
    d = rne_f32(Fraction(float(d1)) + Fraction(float(ph.EPS)))
    if d == 0:
        return F32(np.inf)
    return rne_f32(1 / Fraction(float(d)))


def bits(x):
    return int(np.asarray(x, np.float32).view(np.uint32))


ASSOC_K, ASSOC_RANK = ph.association_case()
K_VALUES = [60.0, 0.0, 1.0, -float(ph.EPS), -3.0, -0.5, float(ASSOC_K), 1e30, 3e38, 3.4e38, -2.5, 7.25, -1e-3, 1e-30]


@pytest.mark.parametrize("k", K_VALUES)
def test_contribution_matches_exact_rounding(k):
    rng = np.random.default_rng(1)
    ranks = sorted(set(range(0, 70)) | set(rng.integers(0, 2048, 200).tolist()) | {1023, 2047})
    for r in ranks:
        got, want = ph.contribution(r, F32(k)), exact_contribution(r, F32(k))
        assert bits(got) == bits(want), (r, k, got, want)


def test_subnormal_and_infinite_contributions():
    c = ph.contribution(0, F32(3e38))
    assert 0 < c < np.finfo(np.float32).tiny          # subnormal, not flushed
    assert bits(c) == bits(exact_contribution(0, F32(3e38)))
    assert ph.contribution(0, F32(-ph.EPS)) == np.inf  # zero denominator
    assert bits(ph.contribution(5, F32(np.inf))) == 0x00000000
    assert bits(ph.contribution(5, F32(-np.inf))) == 0x80000000


def test_sums_match_exact_rounding():
    rng = np.random.default_rng(2)
    for _ in range(2000):
        k = F32(rng.choice([60.0, 0.5, -3.0, 1e30, 3e38, float(ASSOC_K)]))
        a, b = ph.contribution(int(rng.integers(0, 2048)), k), ph.contribution(int(rng.integers(0, 2048)), k)
        if not (np.isfinite(a) and np.isfinite(b)):
            continue
        assert bits(a + b) == bits(rne_f32(Fraction(float(a)) + Fraction(float(b))))


def test_association_case_differs_and_oracle_takes_the_reference_order():
    k, r = ASSOC_K, ASSOC_RANK
    left, right = (F32(r) + k) + ph.EPS, F32(r) + (k + ph.EPS)
    assert left != right
    assert bits(ph.contribution(r, k)) == bits(F32(1.0) / left) != bits(F32(1.0) / right)
    assert bits(ph.contribution(r, k)) == bits(exact_contribution(r, k))
    # never at the default k = 60
    for rank in range(2048):
        assert (F32(rank) + F32(60)) + ph.EPS == F32(rank) + (F32(60) + ph.EPS)


@pytest.mark.parametrize("kbits,want", [(0xFFA00001, 0xFFE00001), (0x7F800001, 0x7FC00001), (0x7FC12345, 0x7FC12345),
                                        (0xFFFFFFFF, 0xFFFFFFFF)])
def test_nan_k_carries_its_payload_quieted(kbits, want):
    k = np.array([kbits], np.uint32).view(np.float32)[0]
    assert bits(ph.contribution(7, k)) == want
    r = ph.fuse([1, 2, 2], [2, 3, 3], k)
    assert [bits(s) for _, s in r] == [want] * 3


def test_single_and_batch_forms_differ_only_for_second_only_keys_at_minus_inf():
    rng = np.random.default_rng(3)
    for k in K_VALUES + [np.inf]:
        for _ in range(30):
            a = rng.integers(0, 40, rng.integers(0, 30)).tolist()
            b = rng.integers(0, 40, rng.integers(0, 30)).tolist()
            x, y = ph.fuse(a, b, k, "batch"), ph.fuse(a, b, k, "single")
            assert [(i, bits(s)) for i, s in x] == [(i, bits(s)) for i, s in y], k
    a, b = [1, 2], [2, 3, 3]
    x = dict((i, bits(s)) for i, s in ph.fuse(a, b, -np.inf, "batch"))
    y = dict((i, bits(s)) for i, s in ph.fuse(a, b, -np.inf, "single"))
    assert x[1] == y[1] == 0x80000000 and x[2] == y[2] == 0x80000000   # keys of the first list: -0 + -0
    assert x[3] == 0x80000000 and y[3] == 0x00000000                     # second list only: or_insert(-0) vs 0.0 + -0.0


def test_first_list_overwrites_second_list_adds():
    k = F32(60)
    c = [ph.contribution(r, k) for r in range(8)]
    r = dict(ph.fuse([7, 8, 7], [9, 9, 7], k))
    assert bits(r[7]) == bits(c[2] + c[2])                 # first list: the worse-ranked 7 wins, then the second adds
    assert bits(r[8]) == bits(c[1])
    assert bits(r[9]) == bits(c[0] + c[1])                 # second list only: or_insert, then +=


def test_no_truncation_and_order():
    rng = np.random.default_rng(4)
    top_k = 10
    a = rng.permutation(1000)[: 3 * top_k].tolist()
    b = rng.permutation(np.arange(1000, 2000))[: 3 * top_k].tolist()
    r = ph.fuse(a, b, 60.0)
    assert len(r) == 6 * top_k                              # disjoint lists: the whole union, not top_k
    keys = [(-ph.total_cmp_key(s), i) for i, s in r]
    assert keys == sorted(keys)
    # equal scores: the smaller id first
    r = ph.fuse([5, 3], [3, 5], 60.0)
    assert [i for i, _ in r] == [3, 5] and bits(r[0][1]) == bits(r[1][1])


def test_replica_ids_collapse_to_one_key():
    r = dict(ph.fuse([12, 13, 20], [12, 21], 60.0, strides=(4, 4)))
    c = [ph.contribution(i, F32(60)) for i in range(3)]
    assert set(r) == {12, 20}
    assert bits(r[12]) == bits(c[1] + c[0])                 # 12 and 13 are replicas of 12: the later one wins, then += 12
    assert bits(r[20]) == bits(c[2] + c[1])


def test_batch_layout():
    ids, scores, counts = ph.fuse_batch(np.array([[1, 2, 0]], np.uint32), [2], np.array([[2, 9]], np.uint32), [1], 60.0)
    assert counts.tolist() == [2] and ids.shape == (1, 5)
    assert ids[0, :2].tolist() == [2, 1] and ids[0, 2:].tolist() == [0xFFFFFFFF] * 3 and not scores[0, 2:].any()
