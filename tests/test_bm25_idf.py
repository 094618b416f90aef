"""The BM25 idf of csrc/bm25_idf.h against the C library, on the host.

The library computes every idf -- a single index's table and a shard group's per-query idf, on the device -- with
bm25_log1pf, the fdlibm algorithm, because the reference's get_idf calls Rust's f32::ln_1p, which is the C library's
log1pf.  That is only right while the two agree bit for bit, so this sweeps every non-negative finite float (the idf
argument is always one) and compares bm25_idf with the log1pf formula on edge and sampled (N, df) pairs.  It is meant to
fail loudly on a machine whose C library's log1pf differs: there the device idf no longer matches the reference.

The driver (tests/bm25_driver.py) is built with g++ under the library's host flags (-O2, no -march) plus -ffp-contract=off
and OpenMP.  tests/test_gpu_bm25_idf.py checks the library's own device and host copies of the header against the same
C library."""
import numpy as np
import pytest

from tests import bm25_driver


@pytest.fixture(scope="module")
def driver():
    if not bm25_driver.GXX:
        pytest.fail("g++ is needed to check bm25_idf.h against the C library's log1pf")
    return bm25_driver.build()


def test_bm25_log1pf_equals_the_c_librarys_log1pf_on_every_non_negative_float(driver):
    out = bm25_driver.run(driver, "sweep").split()
    bad, first = int(out[0]), int(out[1])
    assert bad == 0, (f"bm25_log1pf differs from this C library's log1pf on {bad} inputs, the first at bits {first:#010x}: "
                      "the device idf would not match the reference's f32::ln_1p here")


def idf_pairs():
    big = 0xFFFFFFFF
    edge = [(0, 0), (0, 1), (1, 0), (1, 1), (0, big), (big, 0), (big, big), (big, big - 1), (big - 1, big), (5, 9), (9, 5),
            (1 << 31, 1), (1 << 24, (1 << 24) + 1), ((1 << 24) + 1, 1 << 24), (1000, 999), (1000, 1001), (1 << 20, 1 << 20)]
    rng = np.random.default_rng(17)
    n = rng.integers(0, 1 << 32, 20000, dtype=np.uint64)
    near = (n.astype(np.int64) + rng.integers(-300, 301, n.size)) % (1 << 32)     # df near N, past it (wrapping) too
    small = rng.integers(0, 1 << 12, n.size, dtype=np.uint64)
    sampled = list(zip(n.tolist(), near.tolist())) + list(zip(small.tolist(), rng.integers(0, 1 << 13, n.size).tolist()))
    logn = (2.0 ** rng.uniform(0, 32, 20000)).astype(np.uint64) % (1 << 32)
    sampled += list(zip(logn.tolist(), ((2.0 ** rng.uniform(0, 32, 20000)).astype(np.uint64) % (1 << 32)).tolist()))
    return edge + sampled


def test_bm25_idf_on_edge_and_sampled_pairs(driver):
    pairs = idf_pairs()
    got, want = bm25_driver.pairs(driver, *zip(*pairs))
    assert got.size == len(pairs)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"bm25_idf differs on {bad.size} pairs, the first (N, df) = {pairs[bad[0]]}"
