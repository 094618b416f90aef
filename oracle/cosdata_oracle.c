/*
 * cosdata_oracle.c -- CPU restatement of the cosdata distance / quantization /
 * re-rank arithmetic (the L0 half of the hot path).
 *
 * TEST INFRASTRUCTURE ONLY -- see cosdata_oracle.h.  Compile with
 *   gcc -O3 -mavx2 -mfma -mf16c -ffp-contract=off -fopenmp
 * -ffp-contract=off matters: rustc never contracts `a*b + c` into an FMA, so
 * every scalar loop below must round the product and the sum separately.
 *
 * Reference semantics assumed: release profile (Cargo.toml has no [profile]
 * section => overflow-checks off => integer overflow wraps), x86_64 with
 * AVX2+FMA detected at run time (dot_product.rs:92-157 dispatchers).
 * Rust `as` float->int casts saturate and map NaN to 0.
 */
#include "cosdata_oracle.h"

#include <immintrin.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ helpers */

static inline uint32_t f32_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float bits_f32(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

/* Rust `x as u8` for f32: saturating, NaN -> 0. */
static inline uint8_t rust_f32_as_u8(float x) {
    if (!(x == x)) return 0;
    if (x <= 0.0f) return 0;
    if (x >= 255.0f) return 255;
    return (uint8_t)x; /* truncation toward zero */
}
/* Rust `x as usize` (64-bit) for f32. */
static inline uint64_t rust_f32_as_usize(float x) {
    if (!(x == x)) return 0;
    if (x <= 0.0f) return 0;
    if (x >= 18446744073709551616.0f) return UINT64_MAX;
    return (uint64_t)x;
}
/* Rust f32::max / f32::min: if one operand is NaN the other is returned. */
static inline float rust_fmax(float a, float b) { return (a != a) ? b : ((b != b) ? a : (a > b ? a : b)); }
static inline float rust_fmin(float a, float b) { return (a != a) ? b : ((b != b) ? a : (a < b ? a : b)); }

/* --------------------------------------------------- synthetic data generator
 * Counter-based (splitmix64 finaliser over seed + idx*golden); defined by this
 * repo (include/cosdata_b200.h documents the same formula for the CUDA side).
 * value = (top24 - 2^23) / 2^23, uniform on [-1, 1), exact in f32. */
float orc_synth_value(uint64_t seed, uint64_t idx) {
    uint64_t z = seed + idx * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z = z ^ (z >> 31);
    int32_t m = (int32_t)(z >> 40) - (1 << 23);
    return (float)m * (1.0f / 8388608.0f);
}
void orc_synth_fill(uint64_t seed, uint64_t first_idx, size_t n, float *out) {
    for (size_t i = 0; i < n; ++i) out[i] = orc_synth_value(seed, first_idx + i);
}

/* ------------------------------------------------------------ half (binary16)
 * crate half 2.4.1 `f16::from_f32` (RNE) / `f32::from(f16)`; call sites
 * src/quantization/scalar.rs:40, src/models/dot_product.rs:17.
 * Bit-level software conversion so the result does not depend on F16C. */
uint16_t orc_f32_to_f16(float x) {
    uint32_t u = f32_bits(x);
    uint32_t sign = (u >> 16) & 0x8000u;
    uint32_t e = (u >> 23) & 0xFFu;
    uint32_t m = u & 0x7FFFFFu;
    if (e == 0xFF) { /* inf / nan: half keeps a quiet nan with top mantissa bits */
        if (m == 0) return (uint16_t)(sign | 0x7C00u);
        return (uint16_t)(sign | 0x7C00u | 0x0200u | (m >> 13));
    }
    int32_t exp = (int32_t)e - 127 + 15;
    if (exp >= 31) return (uint16_t)(sign | 0x7C00u); /* overflow -> inf */
    if (exp <= 0) {
        if (exp < -10) return (uint16_t)sign; /* underflow -> signed zero */
        m |= 0x800000u;
        uint32_t shift = (uint32_t)(14 - exp);
        uint32_t half_m = m >> shift;
        uint32_t rem = m & ((1u << shift) - 1u);
        uint32_t halfway = 1u << (shift - 1);
        if (rem > halfway || (rem == halfway && (half_m & 1u))) half_m++;
        return (uint16_t)(sign | half_m);
    }
    uint32_t half = sign | ((uint32_t)exp << 10) | (m >> 13);
    uint32_t rem = m & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (half & 1u))) half++; /* may carry into exponent: correct */
    return (uint16_t)half;
}
float orc_f16_to_f32(uint16_t h) {
    uint32_t sign = ((uint32_t)h & 0x8000u) << 16;
    uint32_t e = (h >> 10) & 0x1Fu;
    uint32_t m = h & 0x3FFu;
    if (e == 0) {
        if (m == 0) return bits_f32(sign);
        /* subnormal: normalise */
        int shift = 0;
        while (!(m & 0x400u)) { m <<= 1; shift++; }
        m &= 0x3FFu;
        return bits_f32(sign | ((uint32_t)(127 - 15 - shift + 1) << 23) | (m << 13));
    }
    if (e == 31) return bits_f32(sign | 0x7F800000u | (m << 13));
    return bits_f32(sign | ((e + 127 - 15) << 23) | (m << 13));
}

/* ------------------------------------------------------------- dot products */

/* src/models/dot_product.rs:9-11 */
uint64_t orc_dot_u8_scalar(const uint8_t *a, const uint8_t *b, size_t n) {
    uint64_t s = 0;
    for (size_t i = 0; i < n; ++i) s += (uint64_t)a[i] * (uint64_t)b[i];
    return s;
}

/* src/models/dot_product/x86_64.rs:68-82 (accumulate_u32) */
static inline uint32_t accumulate_u32(__m256i x) {
    __m256i s1 = _mm256_hadd_epi32(x, x);
    __m256i s2 = _mm256_hadd_epi32(s1, s1);
    __m128i lo = _mm256_castsi256_si128(s2);
    __m128i hi = _mm256_extracti128_si256(s2, 1);
    return (uint32_t)_mm_cvtsi128_si32(_mm_add_epi32(lo, hi));
}

/* src/models/dot_product/x86_64.rs:22-66 */
uint64_t orc_dot_u8_avx2(const uint8_t *a, const uint8_t *b, size_t len) {
    uint64_t dot = 0;
    __m256i sumlo = _mm256_setzero_si256(), sumhi = _mm256_setzero_si256();
    const __m256i zero = _mm256_setzero_si256();
    size_t i = 0;
    while (i + 32 <= len) {
        __m256i va = _mm256_loadu_si256((const __m256i *)(a + i));
        __m256i vb = _mm256_loadu_si256((const __m256i *)(b + i));
        __m256i va_lo = _mm256_unpacklo_epi8(va, zero), va_hi = _mm256_unpackhi_epi8(va, zero);
        __m256i vb_lo = _mm256_unpacklo_epi8(vb, zero), vb_hi = _mm256_unpackhi_epi8(vb, zero);
        sumlo = _mm256_add_epi32(sumlo, _mm256_madd_epi16(va_lo, vb_lo));
        sumhi = _mm256_add_epi32(sumhi, _mm256_madd_epi16(va_hi, vb_hi));
        i += 32;
    }
    dot += (uint64_t)accumulate_u32(sumlo);
    dot += (uint64_t)accumulate_u32(sumhi);
    while (i < len) { dot += (uint64_t)a[i] * (uint64_t)b[i]; i++; }
    return dot;
}

/* src/models/dot_product.rs:13-19 -- scalar, strictly sequential f32 sum, no FMA */
float orc_dot_f16(const uint16_t *a, const uint16_t *b, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) {
        float p = orc_f16_to_f32(a[i]) * orc_f16_to_f32(b[i]);
        s = s + p;
    }
    return s;
}

/* ---- LABELLED EXTENSION (not in the reference): bfloat16 storage, what StorageType::HalfPrecisionFP would compute with
 * half::bf16 in place of half::f16 (BASELINE.json configs[2] says "bf16").  half 2.4 `bf16::from_f32`: round to nearest
 * even on the upper 16 bits, NaN keeps its sign and is quieted. */
uint16_t orc_f32_to_bf16(float v) {
    uint32_t x;
    memcpy(&x, &v, 4);
    if ((x & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((x >> 16) | 0x0040u);
    const uint32_t round_bit = 0x00008000u;
    if ((x & round_bit) != 0 && (x & (3u * round_bit - 1u)) != 0) return (uint16_t)((x >> 16) + 1u);
    return (uint16_t)(x >> 16);
}
float orc_bf16_to_f32(uint16_t h) {
    uint32_t x = (uint32_t)h << 16;
    float f;
    memcpy(&f, &x, 4);
    return f;
}
/* The extension DEFINES its fold step as a fused multiply-add (one rounding): that is what the CUDA kernels compute, and
 * it equals the f16 arm's multiply-then-add whenever the product is a normal f32 -- always for operands quantized from
 * [-1,1] above 1e-19, since two 8-bit significands multiply exactly.  Only f32-subnormal or overflowing products (operands
 * below 1e-19 / above 1e19, which bf16 unlike f16 can hold) would round differently in the two-step form. */
float orc_dot_bf16(const uint16_t *a, const uint16_t *b, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) s = fmaf(orc_bf16_to_f32(a[i]), orc_bf16_to_f32(b[i]), s);
    return s;
}

/* src/models/dot_product.rs:59-62 */
float orc_dot_f32_scalar(const float *a, const float *b, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) {
        float p = a[i] * b[i];
        s = s + p;
    }
    return s;
}

/* src/models/dot_product/x86_64.rs:418-444: 8 FMA lanes, hadd/hadd/lo+hi, scalar tail */
float orc_dot_f32_simd(const float *a, const float *b, size_t n) {
    __m256 sum = _mm256_setzero_ps();
    size_t chunks = n / 8;
    for (size_t i = 0; i < chunks; ++i) {
        __m256 va = _mm256_loadu_ps(a + i * 8);
        __m256 vb = _mm256_loadu_ps(b + i * 8);
        sum = _mm256_fmadd_ps(va, vb, sum);
    }
    __m256 t = _mm256_hadd_ps(sum, sum);
    t = _mm256_hadd_ps(t, t);
    __m128 lo = _mm256_castps256_ps128(t);
    __m128 hi = _mm256_extractf128_ps(t, 1);
    float result = _mm_cvtss_f32(_mm_add_ps(lo, hi));
    for (size_t i = chunks * 8; i < n; ++i) {
        float p = a[i] * b[i];
        result = result + p;
    }
    return result;
}

/* src/models/dot_product/x86_64.rs:190-211 */
static inline uint64_t count_ones_256(__m256i input) {
    const __m256i low_mask = _mm256_set1_epi8(0x0F);
    const __m256i lookup = _mm256_setr_epi8(0, 1, 1, 2, 1, 2, 2, 3, 1, 2, 2, 3, 2, 3, 3, 4,
                                            0, 1, 1, 2, 1, 2, 2, 3, 1, 2, 2, 3, 2, 3, 3, 4);
    __m256i lo = _mm256_and_si256(input, low_mask);
    __m256i hi = _mm256_and_si256(_mm256_srli_epi16(input, 4), low_mask);
    __m256i sum = _mm256_add_epi8(_mm256_shuffle_epi8(lookup, lo), _mm256_shuffle_epi8(lookup, hi));
    __m256i sum16 = _mm256_sad_epu8(sum, _mm256_setzero_si256());
    __m256i sum64 = _mm256_add_epi64(_mm256_unpacklo_epi64(sum16, _mm256_setzero_si256()),
                                     _mm256_unpackhi_epi64(sum16, _mm256_setzero_si256()));
    return (uint64_t)_mm256_extract_epi64(sum64, 0) + (uint64_t)_mm256_extract_epi64(sum64, 2);
}
uint64_t orc_count_ones_256(const uint8_t *p32) {
    return count_ones_256(_mm256_loadu_si256((const __m256i *)p32));
}

/* src/models/dot_product.rs:21-33 */
float orc_dot_binary_scalar(const uint8_t *x, const uint8_t *y, size_t nbytes) {
    uint32_t dp = 0;
    for (size_t i = 0; i < nbytes; ++i) dp += (uint32_t)__builtin_popcount((unsigned)(x[i] & y[i]));
    return (float)dp;
}

/* src/models/dot_product/x86_64.rs:163-187 (note `i + 32 < len`: last block is scalar) */
float orc_dot_binary_avx2(const uint8_t *x, const uint8_t *y, size_t len) {
    uint64_t dp = 0;
    size_t i = 0;
    while (i + 32 < len) {
        __m256i a = _mm256_loadu_si256((const __m256i *)(x + i));
        __m256i b = _mm256_loadu_si256((const __m256i *)(y + i));
        dp += count_ones_256(_mm256_and_si256(a, b));
        i += 32;
    }
    for (; i < len; ++i) dp += (uint64_t)__builtin_popcount((unsigned)(x[i] & y[i]));
    return (float)dp;
}

/* src/models/dot_product.rs:35-57.  x[0..nbytes) is what the reference names
 * "lsb" (plane 0), x[nbytes..2nbytes) "msb" (plane 1). */
float orc_dot_quaternary_scalar(const uint8_t *x, const uint8_t *y, size_t nbytes) {
    const uint8_t *xl = x, *xm = x + nbytes, *yl = y, *ym = y + nbytes;
    uint32_t dp = 0;
    for (size_t i = 0; i < nbytes; ++i) {
        uint32_t lsbs = (uint32_t)__builtin_popcount((unsigned)(xl[i] & yl[i]));
        uint8_t mid1 = xl[i] & ym[i];
        uint8_t mid2 = yl[i] & xm[i];
        uint32_t carry = (uint32_t)__builtin_popcount((unsigned)(mid1 & mid2));
        uint32_t msbs = (uint32_t)__builtin_popcount((unsigned)(xm[i] & ym[i]));
        uint32_t mid = (uint32_t)__builtin_popcount((unsigned)(mid1 ^ mid2));
        dp += (msbs << 2) + (carry << 2) + (mid << 1) + lsbs;
    }
    return (float)dp;
}

/* src/models/dot_product/x86_64.rs:103-160 */
float orc_dot_quaternary_avx2(const uint8_t *x, const uint8_t *y, size_t len) {
    const uint8_t *xl = x, *xm = x + len, *yl = y, *ym = y + len;
    uint64_t dp = 0;
    size_t i = 0;
    while (i + 32 < len) {
        __m256i x_lsb = _mm256_loadu_si256((const __m256i *)(xl + i));
        __m256i x_msb = _mm256_loadu_si256((const __m256i *)(xm + i));
        __m256i y_lsb = _mm256_loadu_si256((const __m256i *)(yl + i));
        __m256i y_msb = _mm256_loadu_si256((const __m256i *)(ym + i));
        __m256i lsbs = _mm256_and_si256(x_lsb, y_lsb);
        __m256i mid1 = _mm256_and_si256(x_lsb, y_msb);
        __m256i mid2 = _mm256_and_si256(y_lsb, x_msb);
        __m256i msbs = _mm256_and_si256(x_msb, y_msb);
        __m256i carry = _mm256_and_si256(mid1, mid2);
        __m256i mid = _mm256_xor_si256(mid1, mid2);
        dp += (count_ones_256(msbs) << 2) + (count_ones_256(carry) << 2) +
              (count_ones_256(mid) << 1) + count_ones_256(lsbs);
        i += 32;
    }
    for (; i < len; ++i) {
        uint32_t lsbs = (uint32_t)__builtin_popcount((unsigned)(xl[i] & yl[i]));
        uint8_t mid1 = xl[i] & ym[i];
        uint8_t mid2 = yl[i] & xm[i];
        uint32_t carry = (uint32_t)__builtin_popcount((unsigned)(mid1 & mid2));
        uint32_t msbs = (uint32_t)__builtin_popcount((unsigned)(xm[i] & ym[i]));
        uint32_t mid = (uint32_t)__builtin_popcount((unsigned)(mid1 ^ mid2));
        dp += (uint64_t)((msbs << 2) + (carry << 2) + (mid << 1) + lsbs);
    }
    return (float)dp;
}

/* src/models/dot_product.rs:64-90: plane 0 "lsb", 1 "mid", 2 "msb" */
float orc_dot_octal_scalar(const uint8_t *x, const uint8_t *y, size_t nbytes) {
    const uint8_t *x0 = x, *x1 = x + nbytes, *x2 = x + 2 * nbytes;
    const uint8_t *y0 = y, *y1 = y + nbytes, *y2 = y + 2 * nbytes;
    uint32_t dp = 0;
    for (size_t i = 0; i < nbytes; ++i) {
        uint32_t sum = 0;
        for (int bit = 0; bit < 8; ++bit) {
            uint32_t xv = (uint32_t)((((x2[i] >> bit) & 1) << 2) | (((x1[i] >> bit) & 1) << 1) | ((x0[i] >> bit) & 1));
            uint32_t yv = (uint32_t)((((y2[i] >> bit) & 1) << 2) | (((y1[i] >> bit) & 1) << 1) | ((y0[i] >> bit) & 1));
            sum += xv * yv;
        }
        dp += sum;
    }
    return (float)dp;
}

/* src/models/dot_product/x86_64.rs:284-407: pack_octal_vectors + 64-entry
 * product LUT via 4x pshufb + blendv; dispatcher src/models/dot_product.rs:135-144 */
static const uint8_t OCTAL_LUT[64] = {
    0, 0, 0, 0, 0, 1, 2, 3, 0, 2, 4, 6, 0, 3, 6, 9,
    0, 0, 0, 0, 4, 5, 6, 7, 8, 10, 12, 14, 12, 15, 18, 21,
    0, 4, 8, 12, 0, 5, 10, 15, 0, 6, 12, 18, 0, 7, 14, 21,
    16, 20, 24, 28, 20, 25, 30, 35, 24, 30, 36, 42, 28, 35, 42, 49};

float orc_dot_octal_avx2(const uint8_t *x, const uint8_t *y, size_t nbytes) {
    const uint8_t *xv[3] = {x, x + nbytes, x + 2 * nbytes};
    const uint8_t *yv[3] = {y, y + nbytes, y + 2 * nbytes};
    size_t n = nbytes * 8;
    uint8_t *data = (uint8_t *)malloc(n ? n : 1);
    for (size_t i = 0; i < nbytes; ++i) {
        for (int j = 0; j < 8; ++j) {
            uint8_t mask = (uint8_t)(1u << j);
            data[i * 8 + j] = (uint8_t)(((yv[0][i] & mask) >> j) | (((yv[1][i] & mask) >> j) << 1) |
                                        (((xv[0][i] & mask) >> j) << 2) | (((xv[1][i] & mask) >> j) << 3) |
                                        (((yv[2][i] & mask) >> j) << 4) | (((xv[2][i] & mask) >> j) << 5));
        }
    }
    const __m256i l0 = _mm256_broadcastsi128_si256(_mm_loadu_si128((const __m128i *)(OCTAL_LUT)));
    const __m256i l1 = _mm256_broadcastsi128_si256(_mm_loadu_si128((const __m128i *)(OCTAL_LUT + 16)));
    const __m256i l2 = _mm256_broadcastsi128_si256(_mm_loadu_si128((const __m128i *)(OCTAL_LUT + 32)));
    const __m256i l3 = _mm256_broadcastsi128_si256(_mm_loadu_si128((const __m128i *)(OCTAL_LUT + 48)));
    const __m256i low_mask = _mm256_set1_epi8(0x0f);
    __m256i acc = _mm256_setzero_si256();
    size_t i = 0;
    while (i + 32 < n) {
        __m256i local = _mm256_setzero_si256();
        for (int rep = 0; rep < 2; ++rep) {
            if (i + 32 >= n) break;
            __m256i vec = _mm256_loadu_si256((const __m256i *)(data + i));
            __m256i vm = _mm256_and_si256(vec, _mm256_set1_epi8(0x3F));
            __m256i lo = _mm256_and_si256(vm, low_mask);
            __m256i hi = _mm256_srli_epi16(vm, 4);
            __m256i r0 = _mm256_shuffle_epi8(l0, lo), r1 = _mm256_shuffle_epi8(l1, lo);
            __m256i r2 = _mm256_shuffle_epi8(l2, lo), r3 = _mm256_shuffle_epi8(l3, lo);
            __m256i b01 = _mm256_blendv_epi8(r0, r1, _mm256_slli_epi16(hi, 7));
            __m256i b23 = _mm256_blendv_epi8(r2, r3, _mm256_slli_epi16(hi, 7));
            __m256i pc = _mm256_blendv_epi8(b01, b23, _mm256_slli_epi16(hi, 6));
            local = _mm256_add_epi8(local, pc);
            i += 32;
        }
        acc = _mm256_add_epi64(acc, _mm256_sad_epu8(local, _mm256_setzero_si256()));
    }
    uint64_t result = 0;
    result += (uint64_t)_mm256_extract_epi64(acc, 0);
    result += (uint64_t)_mm256_extract_epi64(acc, 1);
    result += (uint64_t)_mm256_extract_epi64(acc, 2);
    result += (uint64_t)_mm256_extract_epi64(acc, 3);
    while (i < n) { result += OCTAL_LUT[data[i] & 0x3F]; i++; }
    free(data);
    return (float)result;
}

/* -------------------------------------------------------------- quantization */

size_t orc_code_bytes(int st, size_t dim) {
    switch (st) {
    case ORC_ST_U8: return dim;
    case ORC_ST_SUB1: case ORC_ST_SUB2: case ORC_ST_SUB3: return (size_t)st * ((dim + 7) / 8);
    case ORC_ST_F16: case ORC_ST_BF16: return dim * 2;
    case ORC_ST_F32: return dim * 4;
    default: return 0;
    }
}

/* Rust `iter().map(|x| x*x).sum::<f32>().sqrt()`: sequential left fold from 0.0 */
float orc_mag_f32(const float *v, size_t dim) {
    float s = 0.0f;
    for (size_t i = 0; i < dim; ++i) {
        float p = v[i] * v[i];
        s = s + p;
    }
    return sqrtf(s);
}

/* src/models/common.rs:225-275 (to_float_flag + quantize_to_u8_bits).
 * Plane 0 holds the MOST significant of the low `r` bits of n. */
static void quantize_to_u8_bits(const float *v, size_t dim, unsigned r, uint8_t *out) {
    size_t nbytes = (dim + 7) / 8;
    memset(out, 0, (size_t)r * nbytes);
    float parts = (float)(1u << r);      /* 2_usize.pow(r) as f32 */
    float step = 2.0f / parts;
    for (size_t i = 0; i < dim; ++i) {
        float t = (v[i] + 1.0f) / step;
        uint64_t n = rust_f32_as_usize(floorf(t));
        for (int p = (int)r - 1; p >= 0; --p) { /* result[p] = n&1; n >>= 1 */
            if (n & 1u) out[(size_t)p * nbytes + i / 8] |= (uint8_t)(1u << (i % 8));
            n >>= 1;
        }
    }
}

/* src/quantization/scalar.rs:10-52 */
int orc_quantize(int st, float lo, float hi, const float *v, size_t dim, void *out_code, float *out_mag) {
    switch (st) {
    case ORC_ST_U8: {
        uint8_t *q = (uint8_t *)out_code;
        uint32_t ss = 0; /* u32 sum, wraps in release */
        for (size_t i = 0; i < dim; ++i) {
            float c = rust_fmin(rust_fmax(v[i], lo), hi);
            float t = ((c - lo) / (hi - lo)) * 255.0f;
            q[i] = rust_f32_as_u8(t);
            ss += (uint32_t)q[i] * (uint32_t)q[i];
        }
        *out_mag = sqrtf((float)ss);
        return ORC_OK;
    }
    case ORC_ST_SUB1: case ORC_ST_SUB2: case ORC_ST_SUB3:
        quantize_to_u8_bits(v, dim, (unsigned)st, (uint8_t *)out_code);
        *out_mag = orc_mag_f32(v, dim);
        return ORC_OK;
    case ORC_ST_F16: {
        uint16_t *q = (uint16_t *)out_code;
        for (size_t i = 0; i < dim; ++i) q[i] = orc_f32_to_f16(v[i]);
        *out_mag = orc_mag_f32(v, dim);
        return ORC_OK;
    }
    case ORC_ST_BF16: {
        uint16_t *q = (uint16_t *)out_code;
        for (size_t i = 0; i < dim; ++i) q[i] = orc_f32_to_bf16(v[i]);
        *out_mag = orc_mag_f32(v, dim);
        return ORC_OK;
    }
    case ORC_ST_F32:
        memcpy(out_code, v, dim * 4);
        *out_mag = orc_mag_f32(v, dim);
        return ORC_OK;
    default: return ORC_INVALID;
    }
}

/* -------------------------------------------------------- pairwise distances */

/* src/distance/cosine.rs:223-235 */
static int cosine_from_dot(float dot, float x_mag, float y_mag, float *out) {
    float denom = x_mag * y_mag;
    if (denom == 0.0f) return ORC_CALCULATION_ERROR;
    *out = dot / denom;
    return ORC_OK;
}

/* runtime-dispatched dot (AVX2 path, as on the bench hosts) per storage type;
 * src/distance/cosine.rs:104-216, src/distance/dotproduct.rs:20-63 */
static int storage_dot(int st, size_t dim, const void *x, const void *y, float *dot) {
    size_t nb = (dim + 7) / 8;
    switch (st) {
    case ORC_ST_U8: *dot = (float)orc_dot_u8_avx2((const uint8_t *)x, (const uint8_t *)y, dim); return ORC_OK;
    case ORC_ST_SUB1: *dot = orc_dot_binary_avx2((const uint8_t *)x, (const uint8_t *)y, nb); return ORC_OK;
    case ORC_ST_SUB2: *dot = orc_dot_quaternary_avx2((const uint8_t *)x, (const uint8_t *)y, nb); return ORC_OK;
    case ORC_ST_SUB3: *dot = orc_dot_octal_avx2((const uint8_t *)x, (const uint8_t *)y, nb); return ORC_OK;
    case ORC_ST_F16: *dot = orc_dot_f16((const uint16_t *)x, (const uint16_t *)y, dim); return ORC_OK;
    case ORC_ST_BF16: *dot = orc_dot_bf16((const uint16_t *)x, (const uint16_t *)y, dim); return ORC_OK;
    case ORC_ST_F32: *dot = orc_dot_f32_simd((const float *)x, (const float *)y, dim); return ORC_OK;
    default: return ORC_INVALID;
    }
}

/* src/distance/euclidean.rs:42-53.  `diff * diff` is an i16 multiply: wraps in
 * release for |diff| >= 182 (reproduced as-is). */
static float euclid_u8(const uint8_t *x, const uint8_t *y, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) {
        int16_t diff = (int16_t)((int16_t)x[i] - (int16_t)y[i]);
        int16_t sq = (int16_t)(uint16_t)((uint32_t)((int32_t)diff * (int32_t)diff) & 0xFFFFu);
        s = s + (float)sq;
    }
    return sqrtf(s);
}
/* src/distance/euclidean.rs:55-66 */
static float euclid_f16(const uint16_t *x, const uint16_t *y, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) {
        float d = orc_f16_to_f32(x[i]) - orc_f16_to_f32(y[i]);
        float p = d * d;
        s = s + p;
    }
    return sqrtf(s);
}
/* src/distance/hamming.rs:60-115 */
static float hamming_bytes_masked(const uint8_t *x, const uint8_t *y, size_t n, uint8_t mask) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) s = s + (float)__builtin_popcount((unsigned)((x[i] ^ y[i]) & mask));
    return s;
}
static float hamming_subbyte(const uint8_t *x, const uint8_t *y, size_t nbytes, unsigned r) {
    /* per byte: 8/r fields of r bits => r=3 ignores bits 6..7 (hamming.rs:86-93) */
    uint8_t fieldmask = (uint8_t)((1u << r) - 1u);
    unsigned fields = 8 / r;
    float total = 0.0f;
    for (unsigned p = 0; p < r; ++p) {
        const uint8_t *vx = x + (size_t)p * nbytes, *vy = y + (size_t)p * nbytes;
        for (size_t i = 0; i < nbytes; ++i) {
            for (unsigned f = 0; f < fields; ++f) {
                unsigned shift = f * r;
                uint8_t a = (uint8_t)((vx[i] >> shift) & fieldmask), b = (uint8_t)((vy[i] >> shift) & fieldmask);
                total = total + (float)__builtin_popcount((unsigned)(a ^ b));
            }
        }
    }
    return total;
}
static float euclid_bf16(const uint16_t *x, const uint16_t *y, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) {
        float d = orc_bf16_to_f32(x[i]) - orc_bf16_to_f32(y[i]);
        float p = d * d;
        s = s + p;
    }
    return sqrtf(s);
}
static float hamming_f16(const uint16_t *x, const uint16_t *y, size_t n) {
    float s = 0.0f;
    for (size_t i = 0; i < n; ++i) s = s + (float)__builtin_popcount((unsigned)(x[i] ^ y[i]));
    return s;
}

/* DistanceMetric::calculate (src/models/types.rs:469-495), (Base,Base) arm only
 * (src/distance/cosine.rs:72-74); both sides share one storage type -- a
 * mismatch is reported by the caller as ORC_STORAGE_MISMATCH. */
int orc_distance(int metric, int st, size_t dim, const void *x, float x_mag,
                 const void *y, float y_mag, float *out) {
    size_t nb = (dim + 7) / 8;
    float dot;
    int rc;
    switch (metric) {
    case ORC_METRIC_COSINE:
        rc = storage_dot(st, dim, x, y, &dot);
        if (rc) return rc;
        return cosine_from_dot(dot, x_mag, y_mag, out);
    case ORC_METRIC_DOT:
        if (st == ORC_ST_F32) return ORC_STORAGE_MISMATCH; /* dotproduct.rs:62: no f32 arm */
        rc = storage_dot(st, dim, x, y, &dot);
        if (rc) return rc;
        *out = dot;
        return ORC_OK;
    case ORC_METRIC_EUCLIDEAN:
        switch (st) {
        case ORC_ST_U8: *out = euclid_u8((const uint8_t *)x, (const uint8_t *)y, dim); return ORC_OK;
        case ORC_ST_F16: *out = euclid_f16((const uint16_t *)x, (const uint16_t *)y, dim); return ORC_OK;
        case ORC_ST_BF16: *out = euclid_bf16((const uint16_t *)x, (const uint16_t *)y, dim); return ORC_OK;
        case ORC_ST_SUB1: case ORC_ST_SUB2: case ORC_ST_SUB3: return ORC_UNIMPLEMENTED; /* euclidean.rs:34-37 */
        default: return ORC_STORAGE_MISMATCH;
        }
    case ORC_METRIC_HAMMING:
        switch (st) {
        case ORC_ST_U8: *out = hamming_bytes_masked((const uint8_t *)x, (const uint8_t *)y, dim, 0xFF); return ORC_OK;
        case ORC_ST_SUB1: case ORC_ST_SUB2: case ORC_ST_SUB3:
            *out = hamming_subbyte((const uint8_t *)x, (const uint8_t *)y, nb, (unsigned)st); return ORC_OK;
        case ORC_ST_F16: case ORC_ST_BF16: *out = hamming_f16((const uint16_t *)x, (const uint16_t *)y, dim); return ORC_OK;
        default: return ORC_STORAGE_MISMATCH;
        }
    default: return ORC_INVALID;
    }
}

/* ------------------------------------------------------------------ ordering
 * f32::total_cmp as an unsigned key; MetricResult::cmp reverses it for the
 * distance-like metrics (src/models/types.rs:401-411). */
uint32_t orc_order_key(int metric, float value) {
    uint32_t b = f32_bits(value);
    uint32_t key = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    if (metric == ORC_METRIC_EUCLIDEAN || metric == ORC_METRIC_HAMMING) key = ~key;
    return key;
}

/* -------------------------------------------------- finalize_ann_results math
 * src/vector_store.rs:414-439: cs = dp / (mag_query * mag_raw); no zero check. */
float orc_rerank_cosine(const float *q, float mag_q, const float *v, size_t dim) {
    float dp = orc_dot_f32_simd(q, v, dim);
    float mag_v = orc_mag_f32(v, dim);
    return dp / (mag_q * mag_v);
}

/* ------------------------------------------------------------- top-k helpers */
typedef struct { uint64_t key; } tk_item; /* (order_key << 32) | ~id : larger is better */

static inline uint64_t make_key(uint32_t okey, uint32_t id) { return ((uint64_t)okey << 32) | (uint64_t)(~id); }

/* bounded min-heap on key (root = worst kept) */
typedef struct { uint64_t *h; size_t n, k; } tk_heap;
static void tk_push(tk_heap *t, uint64_t key) {
    uint64_t *h = t->h;
    if (t->n < t->k) {
        size_t i = t->n++;
        h[i] = key;
        while (i > 0) { size_t p = (i - 1) / 2; if (h[p] <= h[i]) break; uint64_t tmp = h[p]; h[p] = h[i]; h[i] = tmp; i = p; }
        return;
    }
    if (t->k == 0 || key <= h[0]) return;
    h[0] = key;
    size_t i = 0;
    for (;;) {
        size_t l = 2 * i + 1, r = l + 1, m = i;
        if (l < t->n && h[l] < h[m]) m = l;
        if (r < t->n && h[r] < h[m]) m = r;
        if (m == i) break;
        uint64_t tmp = h[m]; h[m] = h[i]; h[i] = tmp; i = m;
    }
}
static int cmp_key_desc(const void *a, const void *b) {
    uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
    return (x < y) - (x > y);
}
/* scores travel beside the key through a side table keyed by id */
static void tk_finish(tk_heap *t, int metric, uint32_t *out_ids, float *out_scores, size_t k) {
    qsort(t->h, t->n, sizeof(uint64_t), cmp_key_desc);
    for (size_t i = 0; i < k; ++i) {
        if (i < t->n) {
            uint32_t okey = (uint32_t)(t->h[i] >> 32);
            if (metric == ORC_METRIC_EUCLIDEAN || metric == ORC_METRIC_HAMMING) okey = ~okey;
            uint32_t b = (okey & 0x80000000u) ? (okey & 0x7FFFFFFFu) : ~okey;
            out_ids[i] = ~(uint32_t)(t->h[i] & 0xFFFFFFFFu);
            out_scores[i] = bits_f32(b);
        } else {
            out_ids[i] = 0xFFFFFFFFu;
            out_scores[i] = 0.0f;
        }
    }
}

int orc_brute_topk_f32(const float *corpus, size_t n, size_t dim, const float *queries, size_t nq,
                       size_t k, int threads, uint32_t *out_ids, float *out_scores) {
    if (threads < 1) threads = 1;
    /* norms of stored rows do not depend on the query: computed once per row
       with the same sequential formula finalize_ann_results applies per call */
    float *mags = (float *)malloc(sizeof(float) * (n ? n : 1));
#pragma omp parallel for num_threads(threads) schedule(static)
    for (long long i = 0; i < (long long)n; ++i) mags[i] = orc_mag_f32(corpus + (size_t)i * dim, dim);
    /* one query per worker, like rayon into_par_iter (src/indexes/mod.rs:268) */
#pragma omp parallel for num_threads(threads) schedule(dynamic, 1)
    for (long long qi = 0; qi < (long long)nq; ++qi) {
        const float *q = queries + (size_t)qi * dim;
        float mag_q = orc_mag_f32(q, dim);
        tk_heap t = {(uint64_t *)malloc(sizeof(uint64_t) * (k ? k : 1)), 0, k};
        for (size_t i = 0; i < n; ++i) {
            float dp = orc_dot_f32_simd(q, corpus + i * dim, dim);
            float cs = dp / (mag_q * mags[i]);
            tk_push(&t, make_key(orc_order_key(ORC_METRIC_COSINE, cs), (uint32_t)i));
        }
        tk_finish(&t, ORC_METRIC_COSINE, out_ids + (size_t)qi * k, out_scores + (size_t)qi * k, k);
        free(t.h);
    }
    free(mags);
    return ORC_OK;
}

int orc_brute_topk_codes(int metric, int st, size_t dim, const void *codes, const float *mags, size_t n,
                         const void *qcodes, const float *qmags, size_t nq, size_t k, int threads,
                         uint32_t *out_ids, float *out_scores, uint8_t *err_flags) {
    if (threads < 1) threads = 1;
    size_t cb = orc_code_bytes(st, dim);
    int bad = 0;
#pragma omp parallel for num_threads(threads) schedule(dynamic, 1)
    for (long long qi = 0; qi < (long long)nq; ++qi) {
        const uint8_t *q = (const uint8_t *)qcodes + (size_t)qi * cb;
        tk_heap t = {(uint64_t *)malloc(sizeof(uint64_t) * (k ? k : 1)), 0, k};
        uint8_t err = 0;
        for (size_t i = 0; i < n; ++i) {
            float v;
            int rc = orc_distance(metric, st, dim, q, qmags[qi], (const uint8_t *)codes + i * cb, mags[i], &v);
            if (rc == ORC_CALCULATION_ERROR) { err |= 1; continue; }
            if (rc != ORC_OK) { err |= 2; bad = rc; break; }
            tk_push(&t, make_key(orc_order_key(metric, v), (uint32_t)i));
        }
        if (err_flags) err_flags[qi] = err;
        tk_finish(&t, metric, out_ids + (size_t)qi * k, out_scores + (size_t)qi * k, k);
        free(t.h);
    }
    return bad;
}

/* finalize_ann_results core (src/vector_store.rs:414-443): exact f32 cosine per
 * candidate, sort by total_cmp desc (ties: smaller id first -- oracle rule),
 * truncate k. */
int orc_rerank_f32(const float *corpus, size_t dim, const float *q, const uint32_t *cand, size_t ncand,
                   size_t k, uint32_t *out_ids, float *out_scores) {
    float mag_q = orc_mag_f32(q, dim);
    tk_heap t = {(uint64_t *)malloc(sizeof(uint64_t) * (ncand ? ncand : 1)), 0, ncand};
    for (size_t i = 0; i < ncand; ++i) {
        float cs = orc_rerank_cosine(q, mag_q, corpus + (size_t)cand[i] * dim, dim);
        tk_push(&t, make_key(orc_order_key(ORC_METRIC_COSINE, cs), cand[i]));
    }
    tk_finish(&t, ORC_METRIC_COSINE, out_ids, out_scores, k);
    free(t.h);
    return ORC_OK;
}


/* ------------------------------------------------------------------ value-range sampling
 * sample_embedding (src/indexes/hnsw/mod.rs:202-265): per value, one counter per threshold it exceeds (f32 compares against
 * f32 literals; NaN exceeds nothing).  finalize_sampling (:268-351): percent = (count as f32 / values_count) * 100.0 with
 * values_count = (dimension * embeddings.len()) as f32; first (tightest) threshold with percent <= clamp_margin_percent. */
static const float ORC_SAMPLE_T[7] = {0.025f, 0.05f, 0.1f, 0.2f, 0.3f, 0.4f, 0.5f};

void orc_sample_counts(const float *values, size_t n_values, uint64_t *counts) {
    for (size_t i = 0; i < n_values; ++i) {
        const float v = values[i];
        for (int t = 0; t < 7; ++t) {
            if (v > ORC_SAMPLE_T[t]) counts[t]++;
            if (v < -ORC_SAMPLE_T[t]) counts[7 + t]++;
        }
    }
}

void orc_values_range(const uint64_t *counts, uint64_t n_values, float clamp_margin_percent, float *range) {
    const float values_count = (float)n_values;
    range[0] = -1.0f;
    range[1] = 1.0f;
    for (int t = 0; t < 7; ++t) {
        const float pct = ((float)counts[7 + t] / values_count) * 100.0f;
        if (pct <= clamp_margin_percent) { range[0] = -ORC_SAMPLE_T[t]; break; }
    }
    for (int t = 0; t < 7; ++t) {
        const float pct = ((float)counts[t] / values_count) * 100.0f;
        if (pct <= clamp_margin_percent) { range[1] = ORC_SAMPLE_T[t]; break; }
    }
}
