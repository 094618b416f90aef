// quantize.cu -- ScalarQuantization::quantize (src/quantization/scalar.rs:10-52) and
// quantize_to_u8_bits (src/models/common.rs:225-275) as CUDA kernels, plus the
// on-device synthetic row generator used by the bench (SURVEY.md section 8d).
#include "kernels.h"

namespace cdb {

// Rust `as u8` / `as usize`: saturating, NaN -> 0.
__device__ inline uint32_t rust_as_u8(float x) {
    if (!(x == x) || x <= 0.0f) return 0;
    if (x >= 255.0f) return 255;
    return (uint32_t)x;  // trunc
}
__device__ inline unsigned long long rust_as_usize(float x) {
    if (!(x == x) || x <= 0.0f) return 0;
    if (x >= 18446744073709551616.0f) return 0xFFFFFFFFFFFFFFFFull;
    return (unsigned long long)x;
}
// f32::max / f32::min ignore a NaN operand
__device__ inline float rust_max(float a, float b) { return (a != a) ? b : ((b != b) ? a : (a > b ? a : b)); }
__device__ inline float rust_min(float a, float b) { return (a != a) ? b : ((b != b) ? a : (a < b ? a : b)); }

__device__ inline uint32_t quant_u8(float x, float lo, float hi) {
    float c = rust_min(rust_max(x, lo), hi);
    float t = __fmul_rn(__fdiv_rn(__fsub_rn(c, lo), __fsub_rn(hi, lo)), 255.0f);
    return rust_as_u8(t);
}
// half::f16::from_f32 (scalar.rs:40): round to nearest even; a NaN keeps its sign and top payload bits with the quiet bit
// set, where __float2half_rn would return the canonical 0x7FFF
__device__ inline uint16_t f32_to_f16_bits(float x) {
    const uint32_t u = __float_as_uint(x);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)(((u >> 16) & 0x8000u) | 0x7E00u | ((u & 0x7FFFFFu) >> 13));
    return __half_as_ushort(__float2half_rn(x));
}
// low `r` bits of floor((x+1)/step) (to_float_flag)
__device__ inline uint32_t quant_sub(float x, int r) {
    float step = __fdiv_rn(2.0f, (float)(1u << r));
    float t = floorf(__fdiv_rn(__fadd_rn(x, 1.0f), step));
    return (uint32_t)(rust_as_usize(t) & ((1ull << r) - 1ull));
}

struct SrcMem {
    const float *p;
    uint32_t dim;
    __device__ float get(uint64_t row, uint32_t col) const { return p[row * dim + col]; }
};
struct SrcSynth {
    uint64_t seed;
    uint64_t first_row;
    uint32_t dim;
    __device__ float get(uint64_t row, uint32_t col) const { return synth_value(seed, (first_row + row) * dim + col); }
};

// one thread per 8 consecutive elements of a row
template <class Src>
__global__ void quantize_codes_kernel(Src src, uint64_t n, uint32_t dim, int st, float lo, float hi,
                                      uint8_t *__restrict__ codes, uint32_t row_pitch,
                                      float *__restrict__ raw, uint32_t raw_pitch_elems) {
    const uint32_t groups = (dim + 7) / 8;
    uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= n * groups) return;
    uint64_t row = gid / groups;
    uint32_t g = (uint32_t)(gid % groups);
    uint32_t c0 = g * 8;
    uint32_t cnt = min(8u, dim - c0);
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = (e < (int)cnt) ? src.get(row, c0 + e) : 0.0f;
    uint8_t *out = codes + row * row_pitch;
    if (raw) {
        float *rr = raw + row * raw_pitch_elems + c0;
        for (uint32_t e = 0; e < cnt; ++e) rr[e] = v[e];
    }
    switch (st) {
    case CDB_ST_U8:
        for (uint32_t e = 0; e < cnt; ++e) out[c0 + e] = (uint8_t)quant_u8(v[e], lo, hi);
        break;
    case CDB_ST_SUB1: case CDB_ST_SUB2: case CDB_ST_SUB3: {
        const int r = st;
        const uint32_t pp = plane_pitch(dim);
        uint32_t bytes[3] = {0, 0, 0};
        for (uint32_t e = 0; e < cnt; ++e) {
            uint32_t nbits = quant_sub(v[e], r);
            // plane p holds bit (r-1-p) of n: plane 0 = MSB (common.rs:229-233)
            for (int p = 0; p < r; ++p) bytes[p] |= ((nbits >> (r - 1 - p)) & 1u) << e;
        }
        for (int p = 0; p < r; ++p) out[p * pp + g] = (uint8_t)bytes[p];
        break;
    }
    case CDB_ST_F16: {
        uint16_t *h = reinterpret_cast<uint16_t *>(out) + c0;
        for (uint32_t e = 0; e < cnt; ++e) h[e] = f32_to_f16_bits(v[e]);
        break;
    }
    case CDB_ST_BF16: {
        uint16_t *h = reinterpret_cast<uint16_t *>(out) + c0;
        for (uint32_t e = 0; e < cnt; ++e) h[e] = f32_to_bf16_bits(__float_as_uint(v[e]));
        break;
    }
    case CDB_ST_F32: {
        float *f = reinterpret_cast<float *>(out) + c0;
        for (uint32_t e = 0; e < cnt; ++e) f[e] = v[e];
        break;
    }
    }
}

// one thread per row: the stored magnitude.  u8: sqrt(sum q^2 as u32) of the
// QUANTIZED values (scalar.rs:25-26); all others: sequential f32 fold of the
// ORIGINAL values (scalar.rs:31-32, 41, 45).
template <class Src>
__global__ void mags_kernel(Src src, uint64_t n, uint32_t dim, int st, float lo, float hi, float *__restrict__ mags) {
    uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    if (st == CDB_ST_U8) {
        uint32_t ss = 0;
        for (uint32_t c = 0; c < dim; ++c) {
            uint32_t q = quant_u8(src.get(row, c), lo, hi);
            ss += q * q;
        }
        mags[row] = __fsqrt_rn((float)ss);
    } else {
        float s = 0.0f;
        for (uint32_t c = 0; c < dim; ++c) {
            float x = src.get(row, c);
            s = __fadd_rn(s, __fmul_rn(x, x));
        }
        mags[row] = __fsqrt_rn(s);
    }
}

// Few rows (a query batch): one CTA per row.  The per-row fold is sequential (`iter().map(|x| x*x).sum()`), but the squares
// are produced by the whole CTA with coalesced loads and the chain thread reads them from shared memory -- the
// thread-per-row form above walks global memory element by element (55 us for 1024 x 768 queries, a fixed cost of every
// HNSW / exact search).  u8 magnitudes are a wrapping integer sum: any order.
template <class Src>
__global__ void __launch_bounds__(128) mags_cta_kernel(Src src, uint64_t n, uint32_t dim, int st, float lo, float hi, float *__restrict__ mags) {
    extern __shared__ float sq[];
    __shared__ uint32_t isum;
    const uint64_t row = blockIdx.x;
    const uint32_t tid = threadIdx.x;
    if (st == CDB_ST_U8) {
        if (tid == 0) isum = 0;
        __syncthreads();
        uint32_t ss = 0;
        for (uint32_t c = tid; c < dim; c += 128) {
            const uint32_t q = quant_u8(src.get(row, c), lo, hi);
            ss += q * q;
        }
        atomicAdd(&isum, ss);
        __syncthreads();
        if (tid == 0) mags[row] = __fsqrt_rn((float)isum);
        return;
    }
    for (uint32_t c = tid; c < dim; c += 128) {
        const float x = src.get(row, c);
        sq[c] = __fmul_rn(x, x);
    }
    __syncthreads();
    if (tid == 0) {
        float s = 0.0f;
        for (uint32_t c = 0; c < dim; ++c) s = __fadd_rn(s, sq[c]);
        mags[row] = __fsqrt_rn(s);
    }
}

template <class Src>
static cdb_status run_quantize(Src src, uint64_t n, uint32_t dim, int st, float lo, float hi, uint8_t *codes,
                               uint32_t row_pitch, float *mags, float *raw, uint32_t raw_pitch_elems, cudaStream_t s) {
    if (n == 0) return CDB_OK;
    const uint32_t groups = (dim + 7) / 8;
    uint64_t total = n * groups;
    uint32_t blocks = (uint32_t)((total + 255) / 256);
    quantize_codes_kernel<Src><<<blocks, 256, 0, s>>>(src, n, dim, st, lo, hi, codes, row_pitch, raw, raw_pitch_elems);
    CDB_LAUNCH_CHECK();
    // the squares share the 48 KB default with the kernel's static word (16 bytes with the dynamic area's alignment): at
    // D = 12288 they alone fill it and the launch would fail
    if (n <= 8192 && (size_t)dim * 4 + 16 <= 48 * 1024)
        mags_cta_kernel<Src><<<(uint32_t)n, 128, (size_t)dim * 4, s>>>(src, n, dim, st, lo, hi, mags);
    else
        mags_kernel<Src><<<(uint32_t)((n + 127) / 128), 128, 0, s>>>(src, n, dim, st, lo, hi, mags);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

cdb_status quantize_rows_device(const float *d_vecs, uint64_t n, uint32_t dim, int st, float lo, float hi,
                                uint8_t *d_codes, uint32_t row_pitch, float *d_mags, float *d_raw,
                                uint32_t raw_pitch_elems, cudaStream_t s) {
    return run_quantize(SrcMem{d_vecs, dim}, n, dim, st, lo, hi, d_codes, row_pitch, d_mags, d_raw, raw_pitch_elems, s);
}

cdb_status quantize_rows_synth(uint64_t seed, uint64_t first_row, uint64_t n, uint32_t dim, int st, float lo, float hi,
                               uint8_t *d_codes, uint32_t row_pitch, float *d_mags, float *d_raw,
                               uint32_t raw_pitch_elems, cudaStream_t s) {
    return run_quantize(SrcSynth{seed, first_row, dim}, n, dim, st, lo, hi, d_codes, row_pitch, d_mags, d_raw, raw_pitch_elems, s);
}

// raw-row magnitudes (finalize_ann_results recomputes |v| per call, vector_store.rs:428;
// the value only depends on the row so it is computed once at upload)
__global__ void raw_mags_kernel(const float *__restrict__ raw, uint32_t pitch_elems, uint64_t n, uint32_t dim, float *__restrict__ mags) {
    uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    mags[row] = mag_f32_seq(raw + row * pitch_elems, dim);
}
cdb_status raw_mags_device(const float *d_raw, uint32_t pitch_elems, uint64_t n, uint32_t dim, float *d_mags, cudaStream_t s) {
    if (n == 0) return CDB_OK;
    raw_mags_kernel<<<(uint32_t)((n + 127) / 128), 128, 0, s>>>(d_raw, pitch_elems, n, dim, d_mags);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // namespace cdb
