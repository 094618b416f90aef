// common.cuh -- shared device/host helpers for libcosdata_b200 (sm_90a only).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <string>

#include "../../include/cosdata_b200.h"

namespace cdb {

// ---------------------------------------------------------------- error plumbing
void set_error(const std::string &msg);
extern std::atomic<uint64_t> g_launch_count;

#define CDB_CUDA_TRY(expr)                                                                     \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            ::cdb::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));              \
            return CDB_CUDA_ERROR;                                                             \
        }                                                                                      \
    } while (0)

#define CDB_LAUNCH_CHECK()                                                                     \
    do {                                                                                       \
        ::cdb::g_launch_count.fetch_add(1, std::memory_order_relaxed);                         \
        cudaError_t _e = cudaGetLastError();                                                   \
        if (_e != cudaSuccess) {                                                               \
            ::cdb::set_error(std::string("kernel launch: ") + cudaGetErrorString(_e));         \
            return CDB_CUDA_ERROR;                                                             \
        }                                                                                      \
    } while (0)

// Opt a kernel in to the device's maximum dynamic shared memory ONCE (per device and kernel).  Setting the attribute to
// the size of the launch at hand, as every launch site used to, races when searches run concurrently on one handle: a
// thread lowers the limit between another thread's cudaFuncSetAttribute and its launch ("invalid argument").  The carve-out
// limit does not affect occupancy -- that follows the dynamic size actually requested at launch.
cudaError_t allow_max_dynamic_smem(const void *kernel);
#define CDB_ALLOW_SMEM(kern, bytes)                                                            \
    do {                                                                                       \
        (void)(bytes);                                                                         \
        CDB_CUDA_TRY(::cdb::allow_max_dynamic_smem(reinterpret_cast<const void *>(kern)));     \
    } while (0)

// ---------------------------------------------------------------- layout
// One stored row = code bytes padded to a 16-byte multiple (row_pitch).
//   u8 : D bytes            sub r: r planes of ceil(D/8) bytes, plane p at p*plane_pitch
//   f16: 2D bytes           f32 : 4D bytes
// plane_pitch = ceil(D/8) rounded up to 16 so every plane starts 16B-aligned.
__host__ __device__ inline uint32_t round_up(uint32_t x, uint32_t m) { return (x + m - 1) / m * m; }
__host__ __device__ inline uint32_t plane_bytes(uint32_t dim) { return (dim + 7) / 8; }
__host__ __device__ inline uint32_t plane_pitch(uint32_t dim) { return round_up(plane_bytes(dim), 16); }
__host__ __device__ inline uint32_t row_pitch_bytes(int st, uint32_t dim) {
    switch (st) {
    case CDB_ST_U8: return round_up(dim, 16);
    case CDB_ST_SUB1: case CDB_ST_SUB2: case CDB_ST_SUB3: return (uint32_t)st * plane_pitch(dim);
    case CDB_ST_F16: case CDB_ST_BF16: return round_up(dim * 2, 16);
    case CDB_ST_F32: return round_up(dim * 4, 16);
    default: return 0;
    }
}

// ---------------------------------------------------------------- bfloat16 (labelled extension, CDB_ST_BF16)
// half::bf16::from_f32: round to nearest even on the upper 16 bits; NaN keeps its sign and top payload bits, quiet bit set
__host__ __device__ inline uint16_t f32_to_bf16_bits(uint32_t x) {
    if ((x & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((x >> 16) | 0x0040u);
    const uint32_t round_bit = 0x00008000u;
    if ((x & round_bit) != 0 && (x & (3u * round_bit - 1u)) != 0) return (uint16_t)((x >> 16) + 1u);
    return (uint16_t)(x >> 16);
}

// ---------------------------------------------------------------- ordering
// f32::total_cmp as an unsigned key (MetricResult::cmp, src/models/types.rs:401-411);
// distance-like metrics are reversed so that a larger key is always "better".
__host__ __device__ inline uint32_t order_key(int metric, uint32_t bits) {
    uint32_t key = (bits & 0x80000000u) ? ~bits : (bits | 0x80000000u);
    if (metric == CDB_METRIC_EUCLIDEAN || metric == CDB_METRIC_HAMMING) key = ~key;
    return key;
}
__host__ __device__ inline uint32_t key_to_bits(int metric, uint32_t key) {
    if (metric == CDB_METRIC_EUCLIDEAN || metric == CDB_METRIC_HAMMING) key = ~key;
    return (key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key;
}
// 64-bit selection key: better score first, then smaller id.  0 = empty slot.
__host__ __device__ inline uint64_t make_key64(uint32_t okey, uint32_t id) {
    return ((uint64_t)okey << 32) | (uint64_t)(~id);
}
__host__ __device__ inline uint32_t key64_id(uint64_t k) { return ~(uint32_t)(k & 0xFFFFFFFFull); }

// x86 SSE/AVX produce the "real indefinite" QNaN (sign set) for invalid
// operations such as 0/0; CUDA produces 0x7FFFFFFF.  total_cmp orders the two
// at opposite ends, so results are canonicalised to the reference platform's.
__device__ inline float canon_nan(float v) { return (v != v) ? __uint_as_float(0xFFC00000u) : v; }

// ---------------------------------------------------------------- synthetic data
__host__ __device__ inline float synth_value(uint64_t seed, uint64_t idx) {
    uint64_t z = seed + idx * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    int32_t m = (int32_t)(z >> 40) - (1 << 23);
    return (float)m * (1.0f / 8388608.0f);
}

// ---------------------------------------------------------------- loads
__device__ inline uint4 ldg128(const void *p) { return __ldg(reinterpret_cast<const uint4 *>(p)); }
// streaming load: read-once corpus rows should not pollute L1
__device__ inline uint4 ldg128_stream(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

}  // namespace cdb
