"""The BM25 idf of csrc/bm25_idf.h against the C library, on the host.

The library computes every idf -- a single index's table and a shard group's per-query idf, on the device -- with
bm25_log1pf, the fdlibm algorithm, because the reference's get_idf calls Rust's f32::ln_1p, which is the C library's
log1pf.  That is only right while the two agree bit for bit, so this sweeps every non-negative finite float (the idf
argument is always one) and compares bm25_idf with the log1pf formula on edge and sampled (N, df) pairs.  It is meant to
fail loudly on a machine whose C library's log1pf differs: there the device idf no longer matches the reference.

The driver is built with g++ under the library's host flags (-O2, no -march) plus -ffp-contract=off and OpenMP."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cosdata_b200", "csrc")
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")

DRIVER = r"""
#include <cmath>
#include <cstdio>
#include <cstring>
#include "bm25_idf.h"

static uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

// get_idf as the reference writes it, with the C library's log1pf
static float libc_idf(uint32_t n_docs, uint32_t df) {
    const float num = (float)(uint32_t)(n_docs - df) + 0.5f;
    const float den = (float)df + 0.5f;
    return log1pf(num / den);
}

int main(int argc, char **argv) {
    if (argc > 1 && !strcmp(argv[1], "sweep")) {
        // every non-negative finite float: bits 0 .. 0x7f7fffff
        unsigned long long bad = 0;
        uint32_t first = 0xffffffffu;
        #pragma omp parallel for schedule(static, 1 << 20) reduction(+ : bad)
        for (long long i = 0; i < 0x7f800000LL; ++i) {
            const uint32_t u = (uint32_t)i;
            float x;
            memcpy(&x, &u, 4);
            if (fbits(bm25_log1pf(x)) != fbits(log1pf(x))) {
                ++bad;
                #pragma omp critical
                if (u < first) first = u;
            }
        }
        printf("%llu %u\n", bad, first);
        return 0;
    }
    // pairs: "N df" per line on stdin -> "bm25_idf_bits libc_bits" per line
    unsigned n, d;
    while (scanf("%u %u", &n, &d) == 2) printf("%u %u\n", fbits(bm25_idf(n, d)), fbits(libc_idf(n, d)));
    return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    if not GXX:
        pytest.fail("g++ is needed to check bm25_idf.h against the C library's log1pf")
    d = tmp_path_factory.mktemp("bm25")
    src, exe = d / "driver.cpp", d / "driver"
    src.write_text(DRIVER)
    subprocess.run([GXX, "-O2", "-ffp-contract=off", "-fopenmp", "-I", CSRC, str(src), "-o", str(exe), "-lm"], check=True)
    return str(exe)


def test_bm25_log1pf_equals_the_c_librarys_log1pf_on_every_non_negative_float(driver):
    out = subprocess.run([driver, "sweep"], check=True, capture_output=True, text=True).stdout.split()
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
    inp = "".join(f"{a} {b}\n" for a, b in pairs)
    out = np.array(subprocess.run([driver], input=inp, check=True, capture_output=True, text=True).stdout.split(), np.uint64)
    got, want = out[0::2], out[1::2]
    assert got.size == len(pairs)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"bm25_idf differs on {bad.size} pairs, the first (N, df) = {pairs[bad[0]]}"
