// bm25_idf.h -- the BM25 idf of the TF-IDF index (get_idf, sparse_ann_query.rs:298-302), one definition for the host and
// the device.  Plain C++: g++ compiles it as well as nvcc.
//
// get_idf is log1pf(((N - df) + 0.5) / (df + 0.5)) in f32, with u32 wrapping N - df.  Rust's f32::ln_1p is the platform
// C library's log1pf, which is not correctly rounded, so neither a correctly rounded log1p nor CUDA's log1pf gives its
// bits.  bm25_log1pf is the single-precision fdlibm algorithm (Sun's s_log1pf.c) with the branch thresholds of glibc's
// copy of it (x < 0x3ed413d7 unsplit, mantissa split at 0x3504f7, 2^-29 and 2^-54 for tiny x): on every
// non-negative finite float, a range that holds every argument the idf formula produces, it returns the C library's
// log1pf bit for bit.  tests/test_bm25_idf.py sweeps all 2^31 - 2^23 such floats against the host's log1pf and fails on
// the first difference; tests/test_gpu_bm25_idf.py sweeps them through the library's compiled device copy and checks
// bm25_idf through its device and host copies (cdb_debug_bm25).
//
// Bit identity needs every float operation rounded on its own.  On the device each one is an explicit __f*_rn intrinsic,
// which nvcc never contracts into an FFMA.  On the host the operations are plain: the library's host flags (-O2, no
// -march) target x86-64 without FMA, so nothing is contracted there either.
#pragma once

#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define BM25_HD __host__ __device__
#else
#define BM25_HD
#endif

namespace bm25 {

BM25_HD inline float add(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
BM25_HD inline float sub(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
BM25_HD inline float mul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
BM25_HD inline float div(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
BM25_HD inline float from_i32(int32_t v) {
#if defined(__CUDA_ARCH__)
    return __int2float_rn(v);
#else
    return (float)v;
#endif
}
BM25_HD inline float from_u32(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __uint2float_rn(v);
#else
    return (float)v;
#endif
}
BM25_HD inline int32_t bits(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_int(f);
#else
    int32_t i;
    memcpy(&i, &f, 4);
    return i;
#endif
}
BM25_HD inline float from_bits(int32_t i) {
#if defined(__CUDA_ARCH__)
    return __int_as_float(i);
#else
    float f;
    memcpy(&f, &i, 4);
    return f;
#endif
}

}  // namespace bm25

// log1p(x) for x >= 0 finite: x = 2^k * (1 + f) after the 1 + x split (with a correction term c for the rounding of 1 + x),
// then log(1 + f) = 2s + s * R(s^2), s = f / (2 + f), with fdlibm's degree-7 R (Lp1..Lp7).  Negative, infinite and NaN
// inputs are outside its domain.
BM25_HD inline float bm25_log1pf(float x) {
    using namespace bm25;
    const float ln2_hi = 6.9313812256e-01f;   // 0x3f317180
    const float ln2_lo = 9.0580006145e-06f;   // 0x3717f7d1
    const float Lp1 = 6.6666668653e-01f, Lp2 = 4.0000000596e-01f, Lp3 = 2.8571429849e-01f, Lp4 = 2.2222198546e-01f,
                Lp5 = 1.8183572590e-01f, Lp6 = 1.5313838422e-01f, Lp7 = 1.4798198640e-01f;
    const int32_t hx = bits(x);
    float f = 0.0f, c = 0.0f;
    int32_t k = 1, hu = 0;
    if (hx < 0x3ed413d7) {            // x < sqrt(2) - 1: no split
        if (hx < 0x31000000) {        // x < 2^-29
            if (hx < 0x24800000) return x;   // x < 2^-54
            return sub(x, mul(mul(x, x), 0.5f));
        }
        k = 0;
        f = x;
        hu = 1;
    }
    if (k != 0) {
        float u;
        if (hx < 0x5a000000) {        // x < 2^53: 1 + x is inexact, keep its rounding error in c
            u = add(1.0f, x);
            hu = bits(u);
            k = (hu >> 23) - 127;
            c = k > 0 ? sub(1.0f, sub(u, x)) : sub(x, sub(u, 1.0f));
            c = div(c, u);
        } else {
            u = x;
            hu = bits(u);
            k = (hu >> 23) - 127;
            c = 0.0f;
        }
        hu &= 0x007fffff;
        if (hu < 0x3504f7) {          // mantissa below sqrt(2): u in [1, sqrt(2))
            u = from_bits(hu | 0x3f800000);
        } else {                      // u / 2 in [sqrt(2) / 2, 1)
            k += 1;
            u = from_bits(hu | 0x3f000000);
            hu = (0x00800000 - hu) >> 2;
        }
        f = sub(u, 1.0f);
    }
    const float hfsq = mul(mul(0.5f, f), f);
    const float fk = from_i32(k);
    if (hu == 0) {                    // |f| < 2^-20
        if (f == 0.0f) {
            if (k == 0) return 0.0f;
            c = add(c, mul(fk, ln2_lo));
            return add(mul(fk, ln2_hi), c);
        }
        const float R = mul(hfsq, sub(1.0f, mul(0.66666666666666666f, f)));
        if (k == 0) return sub(f, R);
        return sub(mul(fk, ln2_hi), sub(sub(R, add(c, mul(fk, ln2_lo))), f));
    }
    const float s = div(f, add(2.0f, f));
    const float z = mul(s, s);
    float p = add(Lp6, mul(z, Lp7));   // Lp1 + z * (Lp2 + ... + z * (Lp6 + z * Lp7)), innermost first
    p = add(Lp5, mul(z, p));
    p = add(Lp4, mul(z, p));
    p = add(Lp3, mul(z, p));
    p = add(Lp2, mul(z, p));
    p = add(Lp1, mul(z, p));
    const float R = mul(z, p);
    if (k == 0) return sub(f, sub(hfsq, mul(s, add(hfsq, R))));
    return sub(mul(fk, ln2_hi), sub(sub(hfsq, add(mul(s, add(hfsq, R)), add(c, mul(fk, ln2_lo)))), f));
}

// get_idf: u32 wrapping N - df, round-to-nearest u32 -> f32, + 0.5, divide, log1pf
BM25_HD inline float bm25_idf(uint32_t n_docs, uint32_t df) {
    using namespace bm25;
    const float num = add(from_u32(n_docs - df), 0.5f);
    const float den = add(from_u32(df), 0.5f);
    return bm25_log1pf(div(num, den));
}
