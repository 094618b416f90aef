"""The g++ driver that checks csrc/bm25_idf.h against the C library's log1pf (TEST INFRASTRUCTURE ONLY).

tests/test_bm25_idf.py runs it on the header's g++ build; tests/test_gpu_bm25_idf.py uses its C library side as the reference
for the library's own device and host copies.  Built with g++ under the library's host flags (-O2, no -march) plus
-ffp-contract=off and OpenMP, into a temporary directory keyed by the source's and the header's contents.

Modes (argv[1]):
  sweep                     bm25_log1pf against log1pf on every non-negative finite float -> "bad first_bad_bits"
  branches                  how many of those floats take each branch of bm25_log1pf -> "name count" per line
  sums STRIDE COUNT         log1pf of the floats with bits i * STRIDE, i < COUNT, as one checksum per block of BLOCK
                            indices: sum of (i - block start + 1) * bits(log1pf) mod 2^64 -> one u64 per line
  dump STRIDE FIRST COUNT   the log1pf bits of the floats with bits i * STRIDE, FIRST <= i < FIRST + COUNT, one per line
  (none)                    "N df" pairs on stdin -> "bm25_idf_bits libc_bits" per line, libc_bits being get_idf with log1pf
"""
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cosdata_b200", "csrc")
GXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
FINITE = 0x7F800000        # the non-negative finite floats: bits 0 .. 0x7f7fffff
BLOCK = 1 << 16            # indices per checksum block

SOURCE = r"""
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "bm25_idf.h"

static const unsigned long long BLOCK = 1ull << 16;

static uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static float ffrom(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

// get_idf as the reference writes it, with the C library's log1pf
static float libc_idf(uint32_t n_docs, uint32_t df) {
    const float num = (float)(uint32_t)(n_docs - df) + 0.5f;
    const float den = (float)df + 0.5f;
    return log1pf(num / den);
}

// the branch of bm25_log1pf that x = ffrom(hx) takes, by the header's thresholds:
// 0 x < 2^-54, 1 x < 2^-29, 2 unsplit, 3 split with the mantissa below sqrt(2), 4 at or above it; *hu0: the hu == 0 tail;
// *big: x >= 2^53 (1 + x not formed)
static int branch(uint32_t hx, int *hu0, int *big) {
    *hu0 = *big = 0;
    if (hx < 0x24800000u) return 0;
    if (hx < 0x31000000u) return 1;
    if (hx < 0x3ed413d7u) return 2;
    int32_t hu;
    if (hx < 0x5a000000u) {
        hu = (int32_t)fbits(1.0f + ffrom(hx));
    } else {
        hu = (int32_t)hx;
        *big = 1;
    }
    hu &= 0x007fffff;
    int b = 3;
    if (hu >= 0x3504f7) {
        hu = (0x00800000 - hu) >> 2;
        b = 4;
    }
    *hu0 = hu == 0;
    return b;
}

int main(int argc, char **argv) {
    if (argc > 1 && !strcmp(argv[1], "sweep")) {
        unsigned long long bad = 0;
        uint32_t first = 0xffffffffu;
        #pragma omp parallel for schedule(static, 1 << 20) reduction(+ : bad)
        for (long long i = 0; i < 0x7f800000LL; ++i) {
            const float x = ffrom((uint32_t)i);
            if (fbits(bm25_log1pf(x)) != fbits(log1pf(x))) {
                ++bad;
                #pragma omp critical
                if ((uint32_t)i < first) first = (uint32_t)i;
            }
        }
        printf("%llu %u\n", bad, first);
        return 0;
    }
    if (argc > 1 && !strcmp(argv[1], "branches")) {
        unsigned long long c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c_hu0 = 0, c_big = 0;
        #pragma omp parallel for schedule(static, 1 << 20) reduction(+ : c0, c1, c2, c3, c4, c_hu0, c_big)
        for (long long i = 0; i < 0x7f800000LL; ++i) {
            int hu0, big;
            switch (branch((uint32_t)i, &hu0, &big)) {
            case 0: ++c0; break;
            case 1: ++c1; break;
            case 2: ++c2; break;
            case 3: ++c3; break;
            default: ++c4; break;
            }
            c_hu0 += hu0;
            c_big += big;
        }
        printf("tiny_below_2^-54 %llu\ntiny_below_2^-29 %llu\nunsplit %llu\nsplit_below_sqrt2 %llu\nsplit_at_or_above_sqrt2 %llu\n"
               "hu_zero %llu\nat_least_2^53 %llu\n", c0, c1, c2, c3, c4, c_hu0, c_big);
        return 0;
    }
    if (argc > 3 && !strcmp(argv[1], "sums")) {
        const unsigned long long stride = strtoull(argv[2], 0, 0), count = strtoull(argv[3], 0, 0);
        const long long blocks = (long long)((count + BLOCK - 1) / BLOCK);
        unsigned long long *sum = (unsigned long long *)calloc(blocks ? blocks : 1, 8);
        #pragma omp parallel for schedule(dynamic, 16)
        for (long long b = 0; b < blocks; ++b) {
            unsigned long long s = 0;
            for (unsigned long long i = b * BLOCK; i < (b + 1) * BLOCK && i < count; ++i)
                s += (i - b * BLOCK + 1) * (unsigned long long)fbits(log1pf(ffrom((uint32_t)(i * stride))));
            sum[b] = s;
        }
        for (long long b = 0; b < blocks; ++b) printf("%llu\n", sum[b]);
        free(sum);
        return 0;
    }
    if (argc > 4 && !strcmp(argv[1], "dump")) {
        const unsigned long long stride = strtoull(argv[2], 0, 0), first = strtoull(argv[3], 0, 0), count = strtoull(argv[4], 0, 0);
        for (unsigned long long i = first; i < first + count; ++i) printf("%u\n", fbits(log1pf(ffrom((uint32_t)(i * stride)))));
        return 0;
    }
    unsigned n, d;
    while (scanf("%u %u", &n, &d) == 2) printf("%u %u\n", fbits(bm25_idf(n, d)), fbits(libc_idf(n, d)));
    return 0;
}
"""


def build():
    """-> the driver's path, compiled on first use"""
    if not GXX:
        raise RuntimeError("g++ is needed to check bm25_idf.h against the C library's log1pf")
    with open(os.path.join(CSRC, "bm25_idf.h"), "rb") as f:
        h = hashlib.sha256(SOURCE.encode() + f.read()).hexdigest()[:16]
    exe = os.path.join(tempfile.gettempdir(), f"cdb_bm25_driver_{os.getuid()}_{h}")
    if not os.path.exists(exe):
        d = tempfile.mkdtemp()
        src = os.path.join(d, "driver.cpp")
        with open(src, "w") as f:
            f.write(SOURCE)
        subprocess.run([GXX, "-O2", "-ffp-contract=off", "-fopenmp", "-I", CSRC, src, "-o", exe + f".{os.getpid()}", "-lm"], check=True)
        os.replace(exe + f".{os.getpid()}", exe)
        shutil.rmtree(d, ignore_errors=True)
    return exe


def run(exe, *args, stdin=None):
    return subprocess.run([exe, *map(str, args)], input=stdin, check=True, capture_output=True, text=True).stdout


def pairs(exe, n_docs, df):
    """-> (the header's g++ bm25_idf bits, get_idf with the C library's log1pf bits), u32 each"""
    inp = "".join(f"{a} {b}\n" for a, b in zip(np.asarray(n_docs).tolist(), np.asarray(df).tolist()))
    out = np.array(run(exe, stdin=inp).split(), np.uint64).astype(np.uint32)
    return out[0::2], out[1::2]


def block_sums(bits):
    """the driver's `sums` checksum of u32 bits (numpy), one u64 per block of BLOCK (a short last block included)"""
    b = np.asarray(bits).view(np.uint32).astype(np.uint64)
    pad = (-b.size) % BLOCK
    b = np.concatenate([b, np.zeros(pad, np.uint64)]).reshape(-1, BLOCK)
    return (b * np.arange(1, BLOCK + 1, dtype=np.uint64)).sum(axis=1, dtype=np.uint64)
