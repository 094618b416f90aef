// tensor_scan_u8.cu -- EXACT integer scoring of quantized codes on the tensor cores (S1, BRUTE_CODES,
// configs C4 / the reference's default `UnsignedByte` storage).
//
// dot_product_u8 (src/models/dot_product/x86_64.rs:22-66) and the bit-plane products
// dot_product_binary/quaternary/octal (src/models/dot_product.rs:21-90) are integer contractions
//   sum_i a_i * b_i   with a_i, b_i in 0..255 (u8) or the sub-byte digits 0..1 / 0..3 / 0..7,
// so wgmma .s32.u8.u8 (u8 x u8 -> s32 in registers) computes them bit-exactly: max 255*255*D < 2^31.
// u8 storage is consumed in place; sub-byte storage through an unpacked digit copy (digit =
// plane0 + 2*plane1 + 4*plane2, exactly the weights the reference kernels apply).
//
// The kernel is the KIND = 1 instantiation of tensor_scan_kernel (tensor_scan.cu): same TMA producer, consumer warpgroups,
// bounded-drift CTA groups and the same heap-free class-maximum bound, but on u8 operands and with FINAL scores:
//   DotProduct:  score = dp as f32                       (dotproduct.rs:28,55-60)
//   Cosine:      score = (dp as f32) / (|q| * |row|)     (cosine.rs:120,223-235), 0 denominator -> Err
// Per value one int->float convert (+ one multiply by the row's reciprocal magnitude for cosine) and one FMNMX into the
// class maxima; rows passing the bound are scored exactly and emitted as 64-bit selection keys; select_keys_kernel below
// sorts them and picks the top-k.
#include "kernels.h"
#include "tc_common.cuh"

namespace cdb {

// ------------------------------------------------------------------ final selection: sort the emitted keys
__global__ void __launch_bounds__(256) select_keys_kernel(const uint64_t *__restrict__ cand, const uint32_t *__restrict__ cand_cnt,
                                                          uint32_t cap, int metric, uint32_t k, uint32_t *__restrict__ ids,
                                                          float *__restrict__ scores, uint32_t *__restrict__ counts,
                                                          uint64_t *__restrict__ out_keys) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem);
    const uint32_t q = blockIdx.x, n = min(cand_cnt[q], cap);
    uint32_t P = 1;
    while (P < n) P <<= 1;
    for (uint32_t i = threadIdx.x; i < P; i += blockDim.x) keys[i] = i < n ? cand[(size_t)q * cap + i] : 0ull;
    for (uint32_t j = threadIdx.x; j < k; j += blockDim.x) {
        ids[(size_t)q * k + j] = CDB_INVALID_ID;
        scores[(size_t)q * k + j] = 0.0f;
        if (out_keys) out_keys[(size_t)q * k + j] = 0ull;
    }
    __syncthreads();
    for (uint32_t size = 2; size <= P; size <<= 1)
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t x = keys[lo], y = keys[hi];
                if ((x < y) == desc) { keys[lo] = y; keys[hi] = x; }
            }
            __syncthreads();
        }
    const uint32_t m = min(n, k);
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
        ids[(size_t)q * k + i] = key64_id(keys[i]);
        scores[(size_t)q * k + i] = __uint_as_float(key_to_bits(metric, (uint32_t)(keys[i] >> 32)));
        if (out_keys) out_keys[(size_t)q * k + i] = keys[i];
    }
    if (threadIdx.x == 0 && counts) counts[q] = m;
}

// ------------------------------------------------------------------ sub-byte planes -> u8 digits
// digit = plane0 + 2*plane1 + 4*plane2: the weights dot_product_{binary,quaternary,octal} apply to the planes
__global__ void unpack_digits_kernel(const uint8_t *__restrict__ codes, uint32_t row_pitch, uint64_t n, uint32_t dim, int res,
                                     uint8_t *__restrict__ out, uint32_t out_pitch) {
    const uint32_t nb = plane_bytes(dim), pp = plane_pitch(dim);
    uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= n * nb) return;
    const uint64_t row = gid / nb;
    const uint32_t b = (uint32_t)(gid % nb);
    uint32_t pl[3] = {0, 0, 0};
    for (int p = 0; p < res; ++p) pl[p] = codes[row * row_pitch + (size_t)p * pp + b];
    uint8_t d[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) d[e] = (uint8_t)(((pl[0] >> e) & 1u) | (((pl[1] >> e) & 1u) << 1) | (((pl[2] >> e) & 1u) << 2));
    uint8_t *o = out + row * out_pitch + (size_t)b * 8;
    for (int e = 0; e < 8 && b * 8 + e < dim; ++e) o[e] = d[e];
}

cdb_status unpack_digits_device(const uint8_t *d_codes, uint32_t row_pitch, uint64_t n, uint32_t dim, int res, uint8_t *d_out,
                                uint32_t out_pitch, cudaStream_t s) {
    if (!n) return CDB_OK;
    uint64_t total = n * plane_bytes(dim);
    unpack_digits_kernel<<<(uint32_t)((total + 255) / 256), 256, 0, s>>>(d_codes, row_pitch, n, dim, res, d_out, out_pitch);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// ------------------------------------------------------------------ host
size_t tensor_u8_smem_bytes(uint32_t k) { return tensor_scan_smem_bytes(k); }

// d_x: u8 operand rows [n_rows][pitch] (u8 codes or unpacked digits); d_q: query operand rows padded with zero
// rows to a multiple of 128.  Writes ids/scores/counts (and the packed keys when d_out_keys is given).
cdb_status tensor_u8_scan_device(const uint8_t *d_x, const uint8_t *d_q, uint32_t pitch, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, int metric, const float *d_mags, const float *d_qmags, uint32_t id_base, int *d_gthr,
                                 uint64_t *d_cand, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_err32, uint32_t *d_progress,
                                 uint32_t *d_ids, float *d_scores, uint32_t *d_counts, int sm_count, cudaStream_t s,
                                 uint64_t *d_out_keys) {
    cdb_status rc = tensor_scan_i8_device(d_x, d_q, pitch, n_rows, nq, dim, k, metric, d_mags, d_qmags, id_base, d_gthr, d_cand,
                                          d_cand_cnt, cand_cap, d_err32, d_progress, sm_count, s);
    if (rc) return rc;
    uint32_t P = 1;
    while (P < cand_cap) P <<= 1;
    const size_t ssm = (size_t)P * 8;
    if (ssm > 200 * 1024) { set_error("u8 tensor scan: candidate cap too large for the selection kernel"); return CDB_INVALID_PARAMS; }
    CDB_ALLOW_SMEM(select_keys_kernel, ssm);
    select_keys_kernel<<<nq, 256, ssm, s>>>(d_cand, d_cand_cnt, cand_cap, metric, k, d_ids, d_scores, d_counts, d_out_keys);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // namespace cdb
