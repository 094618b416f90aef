// scorers.cuh -- the reference arithmetic, one (query,row) pair at a time.
//
// Every function reproduces the exact operation order of the reference CPU
// path so that results are bit-identical to it (integer) or to its AVX2
// reduction order (f32).  __fmul_rn/__fadd_rn/__fmaf_rn pin the rounding
// points: rustc never contracts a*b+c, while the AVX2 f32 path uses vfmadd.
//
//   dot_f32   src/models/dot_product/x86_64.rs:418-444  (8 FMA lanes, hadd tree, scalar tail)
//   dot_f16   src/models/dot_product.rs:13-19           (sequential, no FMA)
//   dot_u8    src/models/dot_product/x86_64.rs:22-66    (integer, any order) -> `as f32`
//   binary/quaternary/octal  src/models/dot_product.rs:21-90, x86_64.rs:103-187, 284-407
//   euclid    src/distance/euclidean.rs:42-66
//   hamming   src/distance/hamming.rs:60-115
//   cosine    src/distance/cosine.rs:223-235
#pragma once
#include "common.cuh"

namespace cdb {

// ------------------------------------------------------------------ f32
// single-thread version: lane j of the AVX register is acc[j].  Rows are 16-byte pitched: when both operands are
// 16B-aligned the row is fetched 32 floats at a time (8 independent 128-bit loads in flight) before the FMAs, which
// keep the reference's order (chunk i feeds lane j with element 8i+j).
__device__ inline float dot_f32_avx_order_1t(const float *__restrict__ a, const float *__restrict__ b, uint32_t n) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
    const uint32_t chunks = n / 8;
    uint32_t i = 0;
    if ((((uintptr_t)a | (uintptr_t)b) & 15) == 0) {
        for (; i + 4 <= chunks; i += 4) {
            float4 vb[8], va[8];
#pragma unroll
            for (int t = 0; t < 8; ++t) vb[t] = *reinterpret_cast<const float4 *>(b + 8 * i + 4 * t);
#pragma unroll
            for (int t = 0; t < 8; ++t) va[t] = *reinterpret_cast<const float4 *>(a + 8 * i + 4 * t);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                acc[0] = __fmaf_rn(va[2 * c].x, vb[2 * c].x, acc[0]);
                acc[1] = __fmaf_rn(va[2 * c].y, vb[2 * c].y, acc[1]);
                acc[2] = __fmaf_rn(va[2 * c].z, vb[2 * c].z, acc[2]);
                acc[3] = __fmaf_rn(va[2 * c].w, vb[2 * c].w, acc[3]);
                acc[4] = __fmaf_rn(va[2 * c + 1].x, vb[2 * c + 1].x, acc[4]);
                acc[5] = __fmaf_rn(va[2 * c + 1].y, vb[2 * c + 1].y, acc[5]);
                acc[6] = __fmaf_rn(va[2 * c + 1].z, vb[2 * c + 1].z, acc[6]);
                acc[7] = __fmaf_rn(va[2 * c + 1].w, vb[2 * c + 1].w, acc[7]);
            }
        }
    }
    for (; i < chunks; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = __fmaf_rn(a[8 * i + j], b[8 * i + j], acc[j]);
    }
    float lo = __fadd_rn(__fadd_rn(acc[0], acc[1]), __fadd_rn(acc[2], acc[3]));
    float hi = __fadd_rn(__fadd_rn(acc[4], acc[5]), __fadd_rn(acc[6], acc[7]));
    float r = __fadd_rn(lo, hi);
    for (uint32_t t = chunks * 8; t < n; ++t) r = __fadd_rn(r, __fmul_rn(a[t], b[t]));
    return r;
}

// 8 cooperating threads (consecutive lanes, j = lane & 7): thread j owns AVX
// lane j; the xor-butterfly reproduces ((s0+s1)+(s2+s3))+((s4+s5)+(s6+s7)).
// Every thread of the group returns the full result.
__device__ inline float dot_f32_avx_order_8t(const float *__restrict__ a, const float *__restrict__ b, uint32_t n, int j) {
    float acc = 0.0f;
    uint32_t chunks = n / 8;
    uint32_t i = 0;
    for (; i + 4 <= chunks; i += 4) {
        float a0 = a[8 * i + j], a1 = a[8 * i + 8 + j], a2 = a[8 * i + 16 + j], a3 = a[8 * i + 24 + j];
        float b0 = __ldg(b + 8 * i + j), b1 = __ldg(b + 8 * i + 8 + j), b2 = __ldg(b + 8 * i + 16 + j), b3 = __ldg(b + 8 * i + 24 + j);
        acc = __fmaf_rn(a0, b0, acc);
        acc = __fmaf_rn(a1, b1, acc);
        acc = __fmaf_rn(a2, b2, acc);
        acc = __fmaf_rn(a3, b3, acc);
    }
    for (; i < chunks; ++i) acc = __fmaf_rn(a[8 * i + j], __ldg(b + 8 * i + j), acc);
    acc = __fadd_rn(acc, __shfl_xor_sync(0xFFFFFFFFu, acc, 1));
    acc = __fadd_rn(acc, __shfl_xor_sync(0xFFFFFFFFu, acc, 2));
    acc = __fadd_rn(acc, __shfl_xor_sync(0xFFFFFFFFu, acc, 4));
    for (uint32_t t = chunks * 8; t < n; ++t) acc = __fadd_rn(acc, __fmul_rn(a[t], __ldg(b + t)));
    return acc;
}

// `iter().map(|x| x*x).sum::<f32>().sqrt()` -- sequential left fold (scalar.rs:31,41,45;
// vector_store.rs:412,428)
__device__ inline float mag_f32_seq(const float *__restrict__ v, uint32_t n) {
    float s = 0.0f;
    for (uint32_t i = 0; i < n; ++i) s = __fadd_rn(s, __fmul_rn(v[i], v[i]));
    return __fsqrt_rn(s);
}

// ------------------------------------------------------------------ f16 / bf16 dot products
// The reference's `.sum()` is a sequential left fold of f32(x_i) * f32(y_i).  The product of two halfs (11 + 11 significand
// bits) or two bf16 values (8 + 8) is exact in f32, so s + x*y rounds once -- exactly what a fused multiply-add does: both
// operands are widened exactly (subnormals included; bf16 is the upper half of an f32) and folded with one FFMA per element
// instead of FMUL + FADD; bit-identical (tests: every f16 / bf16 arm against the oracle).
// Rows are 16-byte pitched, so the operands are walked with 128-bit loads; the additions stay strictly in element order.
template <bool BF16>
__device__ __forceinline__ float widen16(uint32_t x, bool hi) {
    if (BF16) return __uint_as_float(hi ? (x & 0xFFFF0000u) : (x << 16));
    return __half2float(__ushort_as_half((unsigned short)(hi ? x >> 16 : x & 0xFFFFu)));
}
template <bool BF16>
__device__ __forceinline__ float fhfma16(float s, uint32_t x, uint32_t y, bool hi) {
    return __fmaf_rn(widen16<BF16>(x, hi), widen16<BF16>(y, hi), s);
}
template <bool BF16>
__device__ __forceinline__ float fhfma16x8(float s, const uint4 &x, const uint4 &y) {
    s = fhfma16<BF16>(s, x.x, y.x, false); s = fhfma16<BF16>(s, x.x, y.x, true);
    s = fhfma16<BF16>(s, x.y, y.y, false); s = fhfma16<BF16>(s, x.y, y.y, true);
    s = fhfma16<BF16>(s, x.z, y.z, false); s = fhfma16<BF16>(s, x.z, y.z, true);
    s = fhfma16<BF16>(s, x.w, y.w, false); s = fhfma16<BF16>(s, x.w, y.w, true);
    return s;
}
template <bool BF16>
__device__ inline float dot16_seq(const uint16_t *__restrict__ a, const uint16_t *__restrict__ b, uint32_t n) {
    float s = 0.0f;
    uint32_t i = 0;
    if ((((uintptr_t)a | (uintptr_t)b) & 15) == 0) {
        for (; i + 64 <= n; i += 64) {   // 64 elements of the stored row in flight at a time
            uint4 vb[8];
#pragma unroll
            for (int t = 0; t < 8; ++t) vb[t] = *reinterpret_cast<const uint4 *>(b + i + 8 * t);
#pragma unroll
            for (int t = 0; t < 8; ++t) s = fhfma16x8<BF16>(s, *reinterpret_cast<const uint4 *>(a + i + 8 * t), vb[t]);
        }
        for (; i + 8 <= n; i += 8)
            s = fhfma16x8<BF16>(s, *reinterpret_cast<const uint4 *>(a + i), *reinterpret_cast<const uint4 *>(b + i));
    }
    for (; i < n; ++i) s = fhfma16<BF16>(s, a[i], b[i], false);
    return s;
}
__device__ inline float dot_f16_seq(const __half *__restrict__ a, const __half *__restrict__ b, uint32_t n) {
    return dot16_seq<false>(reinterpret_cast<const uint16_t *>(a), reinterpret_cast<const uint16_t *>(b), n);
}
// bf16 (labelled extension): same fold
__device__ inline float dot_bf16_seq(const uint16_t *__restrict__ a, const uint16_t *__restrict__ b, uint32_t n) {
    return dot16_seq<true>(a, b, n);
}
__device__ inline float euclid_bf16_seq(const uint16_t *a, const uint16_t *b, uint32_t n) {
    float s = 0.0f;
    for (uint32_t i = 0; i < n; ++i) {
        float d = __fsub_rn(__uint_as_float((uint32_t)a[i] << 16), __uint_as_float((uint32_t)b[i] << 16));
        s = __fadd_rn(s, __fmul_rn(d, d));
    }
    return __fsqrt_rn(s);
}

// ------------------------------------------------------------------ u8
__device__ inline uint64_t dot_u8_int(const uint8_t *__restrict__ a, const uint8_t *__restrict__ b, uint32_t n) {
    uint64_t total = 0;
    uint32_t acc = 0;
    uint32_t i = 0;
    if ((((uintptr_t)a | (uintptr_t)b) & 15) == 0) {
        for (; i + 64 <= n; i += 64) {  // 16 dp4a per block: flush well before u32 could overflow (16384 dp4a)
            uint4 vb[4], va[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) vb[t] = *reinterpret_cast<const uint4 *>(b + i + 16 * t);
#pragma unroll
            for (int t = 0; t < 4; ++t) va[t] = *reinterpret_cast<const uint4 *>(a + i + 16 * t);
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                acc = __dp4a(va[t].x, vb[t].x, acc);
                acc = __dp4a(va[t].y, vb[t].y, acc);
                acc = __dp4a(va[t].z, vb[t].z, acc);
                acc = __dp4a(va[t].w, vb[t].w, acc);
            }
            if ((i & 0xFFC0) == 0xFFC0) { total += acc; acc = 0; }
        }
    }
    // rows are 16B-pitched so 4-byte reads are aligned
    for (; i + 4 <= n; i += 4) {
        uint32_t x = *reinterpret_cast<const uint32_t *>(a + i), y = *reinterpret_cast<const uint32_t *>(b + i);
        acc = __dp4a(x, y, acc);
        if ((i & 0xFFFC) == 0xFFFC) { total += acc; acc = 0; }  // flush before u32 could overflow
    }
    for (; i < n; ++i) acc += (uint32_t)a[i] * (uint32_t)b[i];
    return total + acc;
}

// ------------------------------------------------------------------ sub-byte
// planes at x + p*pp (pp = plane pitch), nb = ceil(D/8) valid bytes per plane.
__device__ inline uint32_t load_word_masked(const uint8_t *p, uint32_t off, uint32_t nb) {
    // 4 bytes at `off`, bytes past nb read as 0 (rows are zero padded, but be explicit)
    uint32_t w = *reinterpret_cast<const uint32_t *>(p + off);
    uint32_t valid = nb - off;
    if (valid < 4) w &= (1u << (8 * valid)) - 1u;
    return w;
}
__device__ inline uint32_t dot_binary_int(const uint8_t *x, const uint8_t *y, uint32_t nb) {
    uint32_t s = 0;
    for (uint32_t off = 0; off < nb; off += 4) s += __popc(load_word_masked(x, off, nb) & load_word_masked(y, off, nb));
    return s;
}
// digit = plane0 + 2*plane1 exactly as dot_product_quaternary weighs them
__device__ inline uint32_t dot_quaternary_int(const uint8_t *x, uint32_t xpp, const uint8_t *y, uint32_t ypp, uint32_t nb) {
    uint32_t s = 0;
    for (uint32_t off = 0; off < nb; off += 4) {
        uint32_t xl = load_word_masked(x, off, nb), xm = load_word_masked(x + xpp, off, nb);
        uint32_t yl = load_word_masked(y, off, nb), ym = load_word_masked(y + ypp, off, nb);
        uint32_t lsbs = xl & yl, msbs = xm & ym, mid1 = xl & ym, mid2 = yl & xm;
        s += ((__popc(msbs) + __popc(mid1 & mid2)) << 2) + (__popc(mid1 ^ mid2) << 1) + __popc(lsbs);
    }
    return s;
}
// digit = plane0 + 2*plane1 + 4*plane2
__device__ inline uint32_t dot_octal_int(const uint8_t *x, uint32_t xpp, const uint8_t *y, uint32_t ypp, uint32_t nb) {
    uint32_t s = 0;
    for (uint32_t off = 0; off < nb; off += 4) {
        uint32_t xv[3], yv[3];
#pragma unroll
        for (int p = 0; p < 3; ++p) { xv[p] = load_word_masked(x + p * xpp, off, nb); yv[p] = load_word_masked(y + p * ypp, off, nb); }
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) s += __popc(xv[i] & yv[j]) << (i + j);
    }
    return s;
}

// ------------------------------------------------------------------ euclid / hamming
__device__ inline float euclid_u8_seq(const uint8_t *a, const uint8_t *b, uint32_t n) {
    float s = 0.0f;
    for (uint32_t i = 0; i < n; ++i) {
        int diff = (int)a[i] - (int)b[i];
        short sq = (short)(unsigned short)((unsigned)(diff * diff) & 0xFFFFu);  // i16 multiply wraps (release build)
        s = __fadd_rn(s, (float)sq);
    }
    return __fsqrt_rn(s);
}
__device__ inline float euclid_f16_seq(const __half *a, const __half *b, uint32_t n) {
    float s = 0.0f;
    for (uint32_t i = 0; i < n; ++i) {
        float d = __fsub_rn(__half2float(a[i]), __half2float(b[i]));
        s = __fadd_rn(s, __fmul_rn(d, d));
    }
    return __fsqrt_rn(s);
}
// all hamming sums are integers < 2^24, so the reference's f32 accumulation is exact
__device__ inline uint32_t hamming_bytes(const uint8_t *a, const uint8_t *b, uint32_t n, uint32_t bytemask4) {
    uint32_t s = 0;
    for (uint32_t off = 0; off < n; off += 4) s += __popc((load_word_masked(a, off, n) ^ load_word_masked(b, off, n)) & bytemask4);
    return s;
}

// ------------------------------------------------------------------ dispatcher
// DistanceMetric::calculate (types.rs:469-495), (Base,Base) arm, single thread.
// x = query side, y = stored row (argument order of vector_store.rs:1186-1187).
// *_pp = plane pitch of that operand (sub-byte only).
__device__ inline int pair_distance(int metric, int st, uint32_t dim,
                                    const void *x, float x_mag, uint32_t x_pp,
                                    const void *y, float y_mag, uint32_t y_pp, float *out) {
    const uint32_t nb = plane_bytes(dim);
    float dot = 0.0f;
    bool have_dot = false;
    if (metric == CDB_METRIC_COSINE || metric == CDB_METRIC_DOT_PRODUCT) {
        switch (st) {
        case CDB_ST_U8: dot = __ull2float_rn(dot_u8_int((const uint8_t *)x, (const uint8_t *)y, dim)); have_dot = true; break;
        case CDB_ST_SUB1: dot = (float)dot_binary_int((const uint8_t *)x, (const uint8_t *)y, nb); have_dot = true; break;
        case CDB_ST_SUB2: dot = (float)dot_quaternary_int((const uint8_t *)x, x_pp, (const uint8_t *)y, y_pp, nb); have_dot = true; break;
        case CDB_ST_SUB3: dot = (float)dot_octal_int((const uint8_t *)x, x_pp, (const uint8_t *)y, y_pp, nb); have_dot = true; break;
        case CDB_ST_F16: dot = dot_f16_seq((const __half *)x, (const __half *)y, dim); have_dot = true; break;
        case CDB_ST_BF16: dot = dot_bf16_seq((const uint16_t *)x, (const uint16_t *)y, dim); have_dot = true; break;
        case CDB_ST_F32:
            if (metric == CDB_METRIC_DOT_PRODUCT) return CDB_STORAGE_MISMATCH;  // dotproduct.rs:62
            dot = dot_f32_avx_order_1t((const float *)x, (const float *)y, dim); have_dot = true; break;
        default: return CDB_INVALID_PARAMS;
        }
    }
    switch (metric) {
    case CDB_METRIC_COSINE: {
        if (!have_dot) return CDB_INVALID_PARAMS;
        float denom = __fmul_rn(x_mag, y_mag);
        if (denom == 0.0f) return CDB_CALCULATION_ERROR;  // cosine.rs:230-231
        *out = canon_nan(__fdiv_rn(dot, denom));
        return CDB_OK;
    }
    case CDB_METRIC_DOT_PRODUCT: *out = dot; return CDB_OK;
    case CDB_METRIC_EUCLIDEAN:
        switch (st) {
        case CDB_ST_U8: *out = canon_nan(euclid_u8_seq((const uint8_t *)x, (const uint8_t *)y, dim)); return CDB_OK;
        case CDB_ST_F16: *out = canon_nan(euclid_f16_seq((const __half *)x, (const __half *)y, dim)); return CDB_OK;
        case CDB_ST_BF16: *out = canon_nan(euclid_bf16_seq((const uint16_t *)x, (const uint16_t *)y, dim)); return CDB_OK;
        case CDB_ST_SUB1: case CDB_ST_SUB2: case CDB_ST_SUB3: return CDB_UNSUPPORTED;  // euclidean.rs:34-37 unimplemented!()
        default: return CDB_STORAGE_MISMATCH;
        }
    case CDB_METRIC_HAMMING:
        switch (st) {
        case CDB_ST_U8: *out = (float)hamming_bytes((const uint8_t *)x, (const uint8_t *)y, dim, 0xFFFFFFFFu); return CDB_OK;
        case CDB_ST_SUB1: case CDB_ST_SUB2: case CDB_ST_SUB3: {
            uint32_t mask = (st == CDB_ST_SUB3) ? 0x3F3F3F3Fu : 0xFFFFFFFFu;  // hamming.rs:86-93: 8/3 = 2 fields
            uint32_t s = 0;
            for (int p = 0; p < st; ++p) s += hamming_bytes((const uint8_t *)x + p * x_pp, (const uint8_t *)y + p * y_pp, nb, mask);
            *out = (float)s;
            return CDB_OK;
        }
        case CDB_ST_F16: case CDB_ST_BF16:
            *out = (float)hamming_bytes((const uint8_t *)x, (const uint8_t *)y, dim * 2, 0xFFFFFFFFu); return CDB_OK;
        default: return CDB_STORAGE_MISMATCH;
        }
    default: return CDB_INVALID_PARAMS;
    }
}

}  // namespace cdb
