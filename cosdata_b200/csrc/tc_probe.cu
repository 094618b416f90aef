// tc_probe.cu -- dense wgmma issue-rate probe: the roofline denominator of the integer tensor path.
//
// tensor_scan_u8.cu computes on wgmma .s32.u8.u8, whose peak has no library yardstick.  This kernel measures it directly:
// every SM keeps one CTA of two warpgroups, each issuing back-to-back M64 x N256 MMAs (K = 32 bytes for u8, 16 halfs for
// f16) on operand tiles that stay resident in shared memory, into its own register accumulator, with no loads, no epilogue,
// no global traffic.  What it reports is the rate the tensor pipe sustains when nothing else limits it -- an upper bound
// for any real kernel (the f16 variant of the probe is printed next to it as a sanity check).
#include <type_traits>

#include "kernels.h"
#include "tc_common.cuh"

namespace cdb {

constexpr uint32_t PR_M = 128, PR_N = 256;
constexpr uint32_t PR_A_BYTES = PR_M * 128, PR_B_BYTES = PR_N * 128;   // one 128-byte swizzle row per matrix row

template <bool I8>
__global__ void __launch_bounds__(256, 1) tc_probe_kernel(uint32_t iters, uint32_t *sink) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    for (uint32_t i = threadIdx.x; i < (PR_A_BYTES + PR_B_BYTES) / 4; i += blockDim.x) reinterpret_cast<uint32_t *>(smem)[i] = 0x01010101u;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes of the tiles -> visible to the MMA's async proxy
    __syncthreads();
    const uint32_t wg = threadIdx.x >> 7;
    const uint32_t sa = smem_u32(smem);
    const uint64_t adesc = make_smem_desc(sa + wg * (PR_A_BYTES / 2)), bdesc = make_smem_desc(sa + PR_A_BYTES);
    using Acc = typename std::conditional<I8, uint32_t, float>::type;
    Acc d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0;
    for (uint32_t it = 0; it < iters; ++it) {
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {   // 4 K-steps of one 128-byte swizzle row
            if constexpr (I8) wgmma_u8(d, adesc + 2 * kk, bdesc + 2 * kk);
            else wgmma_f16(d, adesc + 2 * kk, bdesc + 2 * kk);
        }
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < 128; ++i) {
        if constexpr (I8) x ^= d[i]; else x ^= __float_as_uint(d[i]);
    }
    if (x == 0x9E3779B9u) sink[0] = x;   // keeps the accumulators (and so the MMAs) observable
}

template <bool I8>
static cdb_status run_probe(int sm_count, uint32_t iters, float *ms) {
    auto kern = tc_probe_kernel<I8>;
    const size_t smem = 1024 + PR_A_BYTES + PR_B_BYTES;
    CDB_ALLOW_SMEM(kern, smem);
    cudaEvent_t e0, e1;
    CDB_CUDA_TRY(cudaEventCreate(&e0));
    CDB_CUDA_TRY(cudaEventCreate(&e1));
    uint32_t *sink = nullptr;
    CDB_CUDA_TRY(cudaMalloc(&sink, 4));
    kern<<<sm_count, 256, smem, 0>>>(iters / 8 + 1, sink);   // warm-up
    CDB_LAUNCH_CHECK();
    CDB_CUDA_TRY(cudaEventRecord(e0, 0));
    kern<<<sm_count, 256, smem, 0>>>(iters, sink);
    CDB_LAUNCH_CHECK();
    CDB_CUDA_TRY(cudaEventRecord(e1, 0));
    CDB_CUDA_TRY(cudaEventSynchronize(e1));
    CDB_CUDA_TRY(cudaEventElapsedTime(ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(sink);
    return CDB_OK;
}

}  // namespace cdb

using namespace cdb;

extern "C" cdb_status cdb_debug_tensor_peak(int32_t device, int32_t kind_i8, uint32_t iters, double *out_tops, float *out_ms) {
    if (!out_tops) { set_error("null argument"); return CDB_INVALID_PARAMS; }
    CDB_CUDA_TRY(cudaSetDevice(device));
    int sms = 0;
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    if (!iters) iters = 20000;
    float ms = 0.f;
    cdb_status rc = kind_i8 ? run_probe<true>(sms, iters, &ms) : run_probe<false>(sms, iters, &ms);
    if (rc) return rc;
    const double k_per_mma = kind_i8 ? 32.0 : 16.0;
    const double ops = 2.0 * PR_M * PR_N * k_per_mma * 4.0 * (double)iters * (double)sms;
    *out_tops = ops / ((double)ms / 1000.0) / 1e12;
    if (out_ms) *out_ms = ms;
    return CDB_OK;
}
