// tensor_scan.cu -- wgmma prefilter for the batched brute-force cosine scan (S1, large B).
//
// The dense query x corpus product of configs C2/C5 genuinely is a contraction, so it runs
// on the tensor cores: fp16 copies of the L2-normalised rows ("shadow", built at append time)
// and of the normalised queries are multiplied with wgmma .f32.f16.f16 (fp32 accumulators in
// registers).  The result is an APPROXIMATE cosine a(q,x) with a rigorous error bound eps
// (DESIGN.md section 5); it is used only to discard rows that provably cannot be in the exact top-k:
//     every query keeps the maximum approximate score of each of NG disjoint row classes; the k-th
//     largest class maximum A_k is a lower bound of the k-th best approximate score, so the exact
//     k-th best score is >= A_k - eps, and a row can be in the exact top-k only if a >= A_k - 2*eps.
//     Rows passing that test are appended to the query's candidate list; the class maxima are
//     shared between CTAs through global atomicMax.
// The candidates are then re-scored by rerank_f32_kernel with the reference's exact
// arithmetic, so the final ids/scores are bit-identical to the exact scan.
//
// Kernel anatomy (one CTA per SM, 384 threads):
//   warps 0..7   two consumer warpgroups: wgmma M64 x N256 x K16 on their half of the query tile, accumulators in
//                registers, then the threshold epilogue straight from those registers (setmaxnreg: 232 registers)
//   warps 8..11  producer warpgroup (setmaxnreg: 40 registers), one thread issues the TMA loads:
//                cp.async.bulk.tensor.2d, SWIZZLE_128B, 4-stage mbarrier ring
// Tile: 128 queries (A, K-major) x 256 corpus rows (B, K-major), K block = 64 halfs (128 B).
#include <cstdlib>
#include <type_traits>

#include "kernels.h"
#include "tc_common.cuh"

namespace cdb {

constexpr int TS_BLOCK_M = 128;
constexpr int TS_BLOCK_N = 256;
constexpr int TS_BLOCK_K = 64;  // fp16 elements = one 128-byte swizzle row
constexpr int TS_STAGES = 4;
constexpr int TS_CONSUMERS = 256;                  // two warpgroups of 64 query rows each
constexpr int TS_THREADS = TS_CONSUMERS + 128;     // + the producer warpgroup
constexpr uint32_t TS_A_BYTES = TS_BLOCK_M * TS_BLOCK_K * 2;  // 16 KB
constexpr uint32_t TS_B_BYTES = TS_BLOCK_N * TS_BLOCK_K * 2;  // 32 KB
constexpr uint32_t TS_STAGE_BYTES = TS_A_BYTES + TS_B_BYTES;

struct TensorScanArgs {
    uint64_t n_rows;     // rows visible to this launch (the seeding pass sees a prefix)
    uint32_t n_queries;
    uint32_t k;
    uint32_t kblocks, mtiles, ntiles;
    float two_eps;
    uint32_t id_base;
    uint32_t emit;       // 0: seeding pass (only tightens gthr), 1: emit candidates
    int *ggm;            // [mtiles][64][128] shared class maxima (ordered int, class-major so a tile's queries are
                         // contiguous), init f2ord(-inf)
    uint32_t *cand;      // [n_queries][cand_cap] global ids
    uint32_t *cand_cnt;  // [n_queries]
    uint32_t cand_cap;
    uint32_t *progress;  // [groups] tiles completed by the CTAs of a group (bounded-drift window), zeroed per launch
    uint32_t window;     // a CTA may run at most `window` tiles ahead of the slowest CTA of its group
    uint32_t refresh_mask;  // the shared bound is refreshed when (tile & mask) == mask (and for the first tiles)
    uint32_t has_deg;       // the corpus holds degenerate rows: kernel variant that keeps zero accumulators out of the bound
    // ---- integer form (KIND 1: exact scoring of u8 codes / sub-byte digits on wgmma .s32.u8.u8, tensor_scan_u8.cu)
    int metric;             // CDB_METRIC_COSINE or CDB_METRIC_DOT_PRODUCT
    const float *mags;      // [n_rows] stored magnitudes (cosine)
    const float *qmags;     // [n_queries]
    uint64_t *cand64;       // [n_queries][cand_cap] emitted selection keys (exact scores)
    uint32_t *err32;        // [n_queries] error bits
    float rel;              // threshold = bound * rel - two_eps (1 for the f16 form and for the dot product; 1 - 2^-18 for cosine)
};

// Candidate staging in shared memory: 40 bytes per (consumer thread, query row): slot 0 = count, then 9 row ids (f16 form)
// resp. 4 selection keys (integer form)
constexpr uint32_t TS_STAGE_SLOT_BYTES = 40;
constexpr uint32_t TS_LSTAGE = 9;
constexpr uint32_t TS_KSTAGE = 4;
constexpr int TS_GROUPS = 64;       // at most 64 class maxima per query; the filter supports k <= TS_GROUPS

// rare path: one approximate score passed the threshold -> stage the row id, flush TS_LSTAGE at a time
__device__ __noinline__ void epi_emit(const TensorScanArgs &a, uint32_t qi, uint32_t *stage, uint32_t id) {
    uint32_t c = stage[0];
    stage[1 + c] = id;
    if (++c == TS_LSTAGE) {
        const uint32_t pos = atomicAdd(a.cand_cnt + qi, c);
        for (uint32_t i = 0; i < c; ++i)
            if (pos + i < a.cand_cap) a.cand[(size_t)qi * a.cand_cap + pos + i] = stage[1 + i];
        c = 0;
    }
    stage[0] = c;
}

// integer form: a value passed the filter -> its EXACT score (dp as f32, or dp / (|q| * |row|), cosine.rs:120, 223-235) becomes
// a selection key
__device__ __noinline__ void epi_emit_key(const TensorScanArgs &a, uint32_t qi, uint64_t *stage, int dp, uint64_t row, float qmag) {
    float score = __int2float_rn(dp);   // u64 -> f32 of the reference; dp < 2^31 so the conversion is the same RNE
    if (a.metric == CDB_METRIC_COSINE) {
        const float denom = __fmul_rn(qmag, a.mags[row]);
        if (denom == 0.0f) return;      // Err(CalculationError): flagged per tile / per query in the epilogue, the row is skipped
        score = __fdiv_rn(score, denom);
    }
    uint32_t c = (uint32_t)stage[0];
    stage[1 + c] = make_key64(order_key(a.metric, __float_as_uint(score)), a.id_base + (uint32_t)row);
    if (++c == TS_KSTAGE) {
        const uint32_t pos = atomicAdd(a.cand_cnt + qi, c);
        for (uint32_t i = 0; i < c; ++i)
            if (pos + i < a.cand_cap) a.cand64[(size_t)qi * a.cand_cap + pos + i] = stage[1 + i];
        c = 0;
    }
    stage[0] = c;
}

// bitonic sort of NG register values, descending (fully unrolled: all indices are compile-time)
template <int NG>
__device__ __forceinline__ void sort_desc(float (&v)[NG]) {
#pragma unroll
    for (int size = 2; size <= NG; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
#pragma unroll
            for (int t = 0; t < NG / 2; ++t) {
                const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const float x = v[lo], y = v[hi];
                const float mx = fmaxf(x, y), mn = fminf(x, y);
                v[lo] = desc ? mx : mn;
                v[hi] = desc ? mn : mx;
            }
        }
    }
}

// k-th largest of the NG class maxima of one query (volatile: other CTAs raise them concurrently)
template <int NG>
__device__ __forceinline__ float class_bound(const int *ggm_q, uint32_t k) {
    float g2[NG];
#pragma unroll
    for (int i = 0; i < NG; ++i) g2[i] = ord2f(*reinterpret_cast<const volatile int *>(ggm_q + (size_t)i * TS_BLOCK_M));
    sort_desc<NG>(g2);
    float b = -INFINITY;
#pragma unroll
    for (int i = 0; i < NG; ++i) if ((uint32_t)i == k - 1) b = g2[i];
    return b;
}

// accumulator value -> filter value.  f16 form: the f32 accumulator.  Integer form, dot product: u8 x u8 sums are >= 0, and
// non-negative s32 bit patterns order like non-negative floats (FMNMX and the compare keep denormals), so the raw accumulator
// IS the filter value -- no I2F.  Integer form, cosine: f32(dp) / |row| through the staged reciprocal.
template <int KIND>
__device__ __forceinline__ float acc_value(float x, bool, float) { return x; }
template <int KIND>
__device__ __forceinline__ float acc_value(uint32_t x, bool cosine, float rinv) {
    return cosine ? __int2float_rn((int)x) * rinv : __uint_as_float(x);
}
__device__ __forceinline__ uint32_t acc_bits(float x) { return __float_as_uint(x); }
__device__ __forceinline__ uint32_t acc_bits(uint32_t x) { return x; }

// HAS_DEG: the corpus holds degenerate rows (zero / non-finite / out-of-range norm).  Their shadow rows are all zero, so
// they score a == 0.0f exactly, but their exact score is NaN (worst) or +-inf -- the error bound does not cover them.
// They must not tighten the bound: accumulators that are exactly 0.0f are left out of the class maxima (dropping values
// from a maximum only loosens a lower bound, so a proper row that happens to score 0.0f is harmless).  Degenerate rows
// that are not all-zero are put on every candidate list by the host side (api.cu), all-zero rows are provably worst.
// KIND = 1: the same pipeline on wgmma .s32.u8.u8 (exact): operand rows are 128 BYTES of K per stage (128 u8 elements
// instead of 64 halfs -- identical tile bytes, descriptors and swizzle), and the epilogue's values are exact integer dot
// products: the class-maximum bound works on f32(dp) (dot product) or on f32(dp) / |row| (cosine, the per-row reciprocals
// staged in shared memory per tile), the filter keeps a 2^-18 relative margin for the cosine form and none for the dot
// product, and whatever passes is scored EXACTLY (epi_emit_key) -- final selection keys, not candidates.
//
// Register layout of the epilogue: a consumer thread holds two query rows (r and r + 8 of its warpgroup's 64) and, of each,
// the 64 columns 8j + 2(lane%4) + {0,1}.  Classes are column mod NG, so the thread owns NG/4 classes of each of its queries
// (those = 2(lane%4) or 2(lane%4)+1 mod 8); the four threads of a quad together cover all NG classes of their two queries.
template <int STAGES, int NG, bool HAS_DEG, int KIND>
__global__ void __launch_bounds__(TS_THREADS, 1)
tensor_scan_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_x, TensorScanArgs a) {
    constexpr uint32_t K_ELEMS = KIND == 1 ? 2 * TS_BLOCK_K : TS_BLOCK_K;   // elements per 128-byte row: 128 u8 / 64 halfs
    constexpr int NL = NG / 4;                                              // classes a thread owns per query
    using Acc = typename std::conditional<KIND == 1, uint32_t, float>::type;
    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *tiles = smem;
    uint8_t *lstage = tiles + STAGES * TS_STAGE_BYTES;                                      // [256][2] x 40 bytes
    uint64_t *bars = reinterpret_cast<uint64_t *>(lstage + TS_CONSUMERS * 2 * TS_STAGE_SLOT_BYTES);
    uint64_t *full_bar = bars, *empty_bar = bars + STAGES;
    float *rinv_s = reinterpret_cast<float *>(bars + 2 * STAGES);          // KIND 1 cosine: [2][256] reciprocal row magnitudes
    uint32_t *zflag_s = reinterpret_cast<uint32_t *>(rinv_s + 2 * TS_BLOCK_N);   // [2] a valid row of the tile has |row| = 0

    const int lane = threadIdx.x & 31;

    // work assignment: CTA c owns query tile c % mtiles and every G-th corpus tile
    // gridDim.x is a multiple of mtiles: the mtiles CTAs of group g walk the same corpus tiles g, g+G, ...
    // and are kept within `window` tiles of each other, so a corpus tile is fetched from HBM once and
    // served to the other query tiles from L2.
    const uint32_t mt = blockIdx.x % a.mtiles;
    const uint32_t g = blockIdx.x / a.mtiles;
    const uint32_t G = gridDim.x / a.mtiles;

    if (threadIdx.x == TS_CONSUMERS) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        for (int s = 0; s < STAGES; ++s) { mbar_init(smem_u32(&full_bar[s]), 1); mbar_init(smem_u32(&empty_bar[s]), TS_CONSUMERS / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (threadIdx.x >= TS_CONSUMERS) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (threadIdx.x == TS_CONSUMERS) {
            uint32_t s = 0, phase = 0, t = 0;
            for (uint32_t nt = g; nt < a.ntiles; nt += G, ++t) {
                if (a.mtiles > 1 && t >= a.window) {
                    // bounded drift: every CTA of the group must have consumed tile t - window
                    const uint32_t need = (t - a.window + 1) * a.mtiles;
                    // bounded spin: if a peer CTA is not resident (GPU shared with another stream) we only lose locality
                    for (int spin = 0; spin < 20000 && *reinterpret_cast<volatile uint32_t *>(a.progress + g) < need; ++spin) __nanosleep(64);
                }
                for (uint32_t kb = 0; kb < a.kblocks; ++kb) {
                    mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
                    const uint32_t fb = smem_u32(&full_bar[s]);
                    const uint32_t sa = smem_u32(tiles + (size_t)s * TS_STAGE_BYTES);
                    mbar_expect_tx(fb, TS_STAGE_BYTES);
                    tma_load_2d(sa, &map_q, fb, (int)(kb * K_ELEMS), (int)(mt * TS_BLOCK_M));
                    tma_load_2d(sa + TS_A_BYTES, &map_x, fb, (int)(kb * K_ELEMS), (int)(nt * TS_BLOCK_N));
                    if (++s == STAGES) { s = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumers: MMA + threshold filter =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
        const uint32_t ct = threadIdx.x;                       // 0..255
        const uint32_t wg = ct >> 7, wl = (ct >> 5) & 3, qd = (uint32_t)lane & 3;
        const uint32_t qrow0 = wg * 64 + wl * 16 + ((uint32_t)lane >> 2);   // its two query rows: qrow0, qrow0 + 8
        const bool cosine = KIND == 1 && a.metric == CDB_METRIC_COSINE;
        uint32_t qi[2];
        bool qvalid[2];
        float qmag[2], bound[2], thr[2];
        uint32_t err[2];
        int *ggm_q[2];
        uint32_t *stage[2];
        uint64_t *kstage[2];
        float gm[2][NL];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const uint32_t ql = qrow0 + 8 * i;
            qi[i] = mt * TS_BLOCK_M + ql;
            qvalid[i] = qi[i] < a.n_queries;
            qmag[i] = (KIND == 1 && qvalid[i]) ? a.qmags[qi[i]] : 0.0f;
            err[i] = (cosine && qvalid[i] && qmag[i] == 0.0f && a.n_rows > 0) ? (uint32_t)CDB_ERRFLAG_CALCULATION : 0u;
            ggm_q[i] = a.ggm + (size_t)mt * NG * TS_BLOCK_M + ql;  // + class * 128
            stage[i] = reinterpret_cast<uint32_t *>(lstage + (size_t)(ct * 2 + i) * TS_STAGE_SLOT_BYTES);
            kstage[i] = reinterpret_cast<uint64_t *>(stage[i]);
            if (KIND == 1) kstage[i][0] = 0ull; else stage[i][0] = 0;
#pragma unroll
            for (int l = 0; l < NL; ++l) gm[i][l] = -INFINITY;
            bound[i] = thr[i] = -INFINITY;
            if (qvalid[i]) {  // what earlier launches (the seeding pass) and other CTAs already know
                bound[i] = class_bound<NG>(ggm_q[i], a.k);
                thr[i] = KIND == 1 ? (cosine ? bound[i] * a.rel : bound[i]) : bound[i] - a.two_eps;
            }
        }
        const uint32_t sa0 = smem_u32(tiles);
        uint32_t s = 0, phase = 0, t = 0;
        for (uint32_t nt = g; nt < a.ntiles; nt += G, ++t) {
            const uint64_t row0 = (uint64_t)nt * TS_BLOCK_N;
            const float *rs = rinv_s + (t & 1) * TS_BLOCK_N;
            if (cosine) {
                // reciprocal magnitudes of this tile's rows -> shared memory (double buffered by tile parity); a zero
                // magnitude is an Err for every query that meets the row (cosine.rs:230-231)
                if (ct == 0) zflag_s[t & 1] = 0u;
                asm volatile("bar.sync 1, 256;" ::: "memory");
                const bool valid = row0 + ct < a.n_rows;
                const float mg = valid ? a.mags[row0 + ct] : 0.0f;
                rinv_s[(t & 1) * TS_BLOCK_N + ct] = mg > 0.0f ? __frcp_rn(mg) : 0.0f;
                if (valid && mg == 0.0f) zflag_s[t & 1] = 1u;
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (zflag_s[t & 1]) {
#pragma unroll
                    for (int i = 0; i < 2; ++i) if (qvalid[i]) err[i] |= (uint32_t)CDB_ERRFLAG_CALCULATION;
                }
            }
            // ---- the tile's product: kblocks x 4 wgmma into registers; a stage is released when its MMAs have retired
            Acc acc[128];
#pragma unroll
            for (int i = 0; i < 128; ++i) acc[i] = 0;
            uint32_t prev = 0;
            for (uint32_t kb = 0; kb < a.kblocks; ++kb) {
                mbar_wait(smem_u32(&full_bar[s]), phase);
                const uint32_t sa = sa0 + s * TS_STAGE_BYTES;
                const uint64_t adesc = make_smem_desc(sa + wg * (TS_A_BYTES / 2)), bdesc = make_smem_desc(sa + TS_A_BYTES);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {  // +32 bytes along K = +2 in the encoded start address
                    if constexpr (KIND == 1) wgmma_u8(acc, adesc + 2 * kk, bdesc + 2 * kk);
                    else wgmma_f16(acc, adesc + 2 * kk, bdesc + 2 * kk);
                }
                wgmma_commit();
                wgmma_wait<1>();                                   // the previous k-block's MMAs have retired
                if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
                prev = s;
                if (++s == STAGES) { s = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            if (a.kblocks > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
            if (ct == 0 && a.mtiles > 1) atomicAdd(a.progress + g, 1u);   // all loads of this tile have landed in smem

            // ---- epilogue: fold the values into the class maxima, test the tile maximum against the threshold,
            //      build the per-value tests only on a hit
            const bool full_tile = row0 + TS_BLOCK_N <= a.n_rows;   // only the corpus' last tile can be partial (TMA zero fill)
            const uint64_t left = a.n_rows > row0 ? a.n_rows - row0 : 0;   // valid columns of this tile
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                bool hit;
                if (full_tile) {
                    float cm[NL];
#pragma unroll
                    for (int l = 0; l < NL; ++l) cm[l] = -INFINITY;
                    float zmax = -INFINITY;   // HAS_DEG: 0.0f if some accumulator of the tile is exactly zero
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
#pragma unroll
                        for (int b = 0; b < 2; ++b) {
                            const uint32_t col = 8 * j + 2 * qd + b;
                            float v = acc_value<KIND>(acc[4 * j + 2 * i + b], cosine, cosine ? rs[col] : 0.0f);
                            if (HAS_DEG) {
                                zmax = v == 0.0f ? 0.0f : zmax;
                                v = v == 0.0f ? -INFINITY : v;
                            }
                            const int l = (j & (NG / 8 - 1)) * 2 + b;
                            cm[l] = fmaxf(cm[l], v);
                        }
                    }
                    float cmax = zmax;   // the emission test sees every value, the bound only the non-zero ones
#pragma unroll
                    for (int l = 0; l < NL; ++l) { cmax = fmaxf(cmax, cm[l]); gm[i][l] = fmaxf(gm[i][l], cm[l]); }
                    hit = cmax >= thr[i];
                } else {
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
#pragma unroll
                        for (int b = 0; b < 2; ++b) {
                            const uint32_t col = 8 * j + 2 * qd + b;
                            const float v = acc_value<KIND>(acc[4 * j + 2 * i + b], cosine, cosine ? rs[col] : 0.0f);
                            const int l = (j & (NG / 8 - 1)) * 2 + b;
                            if ((uint64_t)col < left && !(HAS_DEG && v == 0.0f)) gm[i][l] = fmaxf(gm[i][l], v);
                        }
                    }
                    hit = true;
                }
                if (qvalid[i] && a.emit && hit) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
#pragma unroll
                        for (int b = 0; b < 2; ++b) {
                            const uint32_t col = 8 * j + 2 * qd + b;
                            const float v = acc_value<KIND>(acc[4 * j + 2 * i + b], cosine, cosine ? rs[col] : 0.0f);
                            if ((uint64_t)col < left && v >= thr[i]) {
                                if (KIND == 1) epi_emit_key(a, qi[i], kstage[i], (int)acc_bits(acc[4 * j + 2 * i + b]), row0 + col, qmag[i]);
                                else epi_emit(a, qi[i], stage[i], a.id_base + (uint32_t)(row0 + col));
                            }
                        }
                    }
                }
            }
            // refresh the shared bound: every tile early on (and in the seeding pass), then every 16th tile.  The quad's
            // classes are published before any of its threads reads the maxima back.
            if (t < 8 || (t & a.refresh_mask) == a.refresh_mask || !a.emit) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    if (!qvalid[i]) continue;
#pragma unroll
                    for (int l = 0; l < NL; ++l) {
                        int *p = ggm_q[i] + (size_t)(8 * (l >> 1) + 2 * qd + (l & 1)) * TS_BLOCK_M;
                        const int mine = f2ord(gm[i][l]);
                        if (mine > *reinterpret_cast<volatile int *>(p)) atomicMax(p, mine);
                    }
                }
                __syncwarp();
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    if (!qvalid[i]) continue;
                    const float nb = class_bound<NG>(ggm_q[i], a.k);
                    if (nb > bound[i]) { bound[i] = nb; thr[i] = KIND == 1 ? (cosine ? bound[i] * a.rel : bound[i]) : bound[i] - a.two_eps; }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!qvalid[i]) continue;
            // final publish + flush of the staged candidates
#pragma unroll
            for (int l = 0; l < NL; ++l) atomicMax(ggm_q[i] + (size_t)(8 * (l >> 1) + 2 * qd + (l & 1)) * TS_BLOCK_M, f2ord(gm[i][l]));
            const uint32_t c = KIND == 1 ? (uint32_t)kstage[i][0] : stage[i][0];
            if (a.emit && c) {
                const uint32_t pos = atomicAdd(a.cand_cnt + qi[i], c);
                for (uint32_t x = 0; x < c; ++x)
                    if (pos + x < a.cand_cap) {
                        if (KIND == 1) a.cand64[(size_t)qi[i] * a.cand_cap + pos + x] = kstage[i][1 + x];
                        else a.cand[(size_t)qi[i] * a.cand_cap + pos + x] = stage[i][1 + x];
                    }
            }
            if (KIND == 1 && err[i]) atomicOr(a.err32 + qi[i], err[i]);
        }
    }
}

// ------------------------------------------------------------------ fp16 normalised copies
// x_hat = x / |x| (IEEE), rounded to fp16.  Rows whose norm is outside [1e-15, 1e15] (zero, underflowed, overflowed,
// inf/NaN) are DEGENERATE: the error bound of the prefilter does not cover them, their shadow row is all zero.
__host__ __device__ inline bool norm_is_proper(float m) { return m >= 1.0e-15f && m <= 1.0e15f; }

__global__ void normalize_f16_kernel(const float *__restrict__ raw, uint32_t pitch_elems, const float *__restrict__ mags,
                                     uint64_t n, uint32_t dim, __half *__restrict__ out, uint32_t out_pitch) {
    const uint32_t groups = (dim + 7) / 8;
    uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= n * groups) return;
    uint64_t row = gid / groups;
    uint32_t c0 = (uint32_t)(gid % groups) * 8;
    const float m = mags[row];
    const bool ok = norm_is_proper(m);
    for (uint32_t e = 0; e < 8 && c0 + e < dim; ++e) {
        float v = raw[row * pitch_elems + c0 + e];
        out[row * out_pitch + c0 + e] = __float2half_rn(ok ? __fdiv_rn(v, m) : 0.0f);
    }
}

cdb_status normalize_f16_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t n, uint32_t dim,
                                void *d_out, uint32_t out_pitch_halfs, cudaStream_t s) {
    if (!n) return CDB_OK;
    uint64_t total = n * ((dim + 7) / 8);
    normalize_f16_kernel<<<(uint32_t)((total + 255) / 256), 256, 0, s>>>(d_raw, pitch_elems, d_mags, n, dim,
                                                                          reinterpret_cast<__half *>(d_out), out_pitch_halfs);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// Degenerate rows of an appended range.  deg = {all-zero rows, other degenerate rows, ids of the first TS_MAX_ODD of those}.
// An all-zero row scores 0/0 = NaN against every finite query: provably last.  Any other degenerate row (norm underflowed
// to 0 with non-zero elements -> +-inf, overflowed norm -> 0 or NaN, inf/NaN elements) can land anywhere in the exact
// ranking, so those rows are put on every query's candidate list and re-scored exactly.
__global__ void classify_rows_kernel(const float *__restrict__ raw, uint32_t pitch_elems, const float *__restrict__ mags,
                                     uint64_t n, uint32_t dim, uint32_t first_row, uint32_t *deg) {
    const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    if (norm_is_proper(mags[row])) return;
    bool allzero = true;
    for (uint32_t c = 0; c < dim && allzero; ++c) allzero = raw[row * pitch_elems + c] == 0.0f;
    if (allzero) { atomicAdd(deg, 1u); return; }
    const uint32_t pos = atomicAdd(deg + 1, 1u);
    if (pos < TS_MAX_ODD) deg[2 + pos] = first_row + (uint32_t)row;
}
cdb_status classify_rows_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t n, uint32_t dim,
                                uint32_t first_row, uint32_t *d_deg, cudaStream_t s) {
    if (!n) return CDB_OK;
    classify_rows_kernel<<<(uint32_t)((n + 255) / 256), 256, 0, s>>>(d_raw, pitch_elems, d_mags, n, dim, first_row, d_deg);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// One launch prepares everything a prefilter search needs from the raw query batch (it replaces eleven memsets / small
// kernels whose launch gaps were a fixed ~0.1 ms per batch -- the limiter of strong scaling once the scan itself takes 1.6 ms):
//   q_raw   f32 copy in the index's pitched layout (operand of the exact re-rank), zero padded
//   q_mags  |q| = sqrt of the SEQUENTIAL fold of x*x (vector_store.rs:412), one thread, squares staged in shared memory
//   qh      fp16 copy of q / |q| (zero row for a degenerate norm and for the padding rows up to mtiles*128)
//   ggm     class maxima of the query := -inf;  cand_cnt := number of pre-seeded odd rows (+ their ids);  err := 0
//   progress counters of the seeding and of the main pass := 0
// One CTA of 128 threads per query slot (mtiles*128 slots).
__global__ void __launch_bounds__(128) prep_queries_kernel(const float *__restrict__ q, uint32_t nq, uint32_t dim, float *__restrict__ q_raw,
                                                           uint32_t raw_pitch_elems, float *__restrict__ q_mags, __half *__restrict__ qh,
                                                           uint32_t qh_pitch, int *__restrict__ ggm, const uint32_t *__restrict__ deg,
                                                           uint32_t has_deg, uint32_t id_base, uint32_t *__restrict__ cand,
                                                           uint32_t cand_cap, uint32_t *__restrict__ cand_cnt, uint32_t *__restrict__ err32,
                                                           uint8_t *__restrict__ err8, uint32_t *__restrict__ progress) {
    extern __shared__ float sq[];     // [dim] squares
    __shared__ float s_mag;
    const uint32_t slot = blockIdx.x, tid = threadIdx.x;
    if (slot == 0) for (uint32_t i = tid; i < 2048; i += 128) progress[i] = 0u;
    // class maxima: layout [tile][class][128]
    if (tid < (uint32_t)TS_GROUPS) ggm[((size_t)(slot >> 7) * TS_GROUPS + tid) * TS_BLOCK_M + (slot & 127u)] = (int)0x807FFFFF;   // f2ord(-inf)
    __half *hrow = qh + (size_t)slot * qh_pitch;
    if (slot >= nq) {
        for (uint32_t c = tid; c < qh_pitch; c += 128) hrow[c] = __float2half_rn(0.0f);
        return;
    }
    const float *src = q + (size_t)slot * dim;
    float *dst = q_raw + (size_t)slot * raw_pitch_elems;
    for (uint32_t c = tid; c < raw_pitch_elems; c += 128) {
        const float v = c < dim ? src[c] : 0.0f;
        dst[c] = v;
        if (c < dim) sq[c] = __fmul_rn(v, v);
    }
    __syncthreads();
    if (tid == 0) {
        float s = 0.0f;
        for (uint32_t c = 0; c < dim; ++c) s = __fadd_rn(s, sq[c]);
        const float m = __fsqrt_rn(s);
        s_mag = m;
        q_mags[slot] = m;
        err32[slot] = 0u;
        if (err8) err8[slot] = 0;
        uint32_t n_odd = 0;
        if (has_deg) {
            n_odd = min(min(deg[1], (uint32_t)TS_MAX_ODD), cand_cap);
            for (uint32_t i = 0; i < n_odd; ++i) cand[(size_t)slot * cand_cap + i] = id_base + deg[2 + i];
        }
        cand_cnt[slot] = n_odd;
    }
    __syncthreads();
    const float m = s_mag;
    const bool ok = norm_is_proper(m);
    for (uint32_t c = tid; c < qh_pitch; c += 128)
        hrow[c] = __float2half_rn((ok && c < dim) ? __fdiv_rn(src[c], m) : 0.0f);
}

cdb_status prep_queries_device(const float *d_q, uint32_t nq, uint32_t dim, float *d_q_raw, uint32_t raw_pitch_elems, float *d_q_mags,
                               void *d_qh, uint32_t qh_pitch_halfs, int *d_ggm, const uint32_t *d_deg, bool has_deg, uint32_t id_base,
                               uint32_t *d_cand, uint32_t cand_cap, uint32_t *d_cand_cnt, uint32_t *d_err32, uint8_t *d_err8,
                               uint32_t *d_progress, cudaStream_t s) {
    const uint32_t mtiles = (nq + TS_BLOCK_M - 1) / TS_BLOCK_M;
    prep_queries_kernel<<<mtiles * TS_BLOCK_M, 128, (size_t)dim * 4, s>>>(d_q, nq, dim, d_q_raw, raw_pitch_elems, d_q_mags,
                                                                          reinterpret_cast<__half *>(d_qh), qh_pitch_halfs, d_ggm, d_deg,
                                                                          has_deg ? 1u : 0u, id_base, d_cand, cand_cap, d_cand_cnt, d_err32,
                                                                          d_err8, d_progress);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// candidate lists start with the odd degenerate rows (global ids); cand_cnt[q] = n_odd
__global__ void seed_candidates_kernel(const uint32_t *__restrict__ deg, uint32_t id_base, uint32_t nq, uint32_t *cand,
                                       uint32_t cand_cap, uint32_t *cand_cnt) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    const uint32_t n_odd = min(min(deg[1], (uint32_t)TS_MAX_ODD), cand_cap);
    for (uint32_t i = 0; i < n_odd; ++i) cand[(size_t)q * cand_cap + i] = id_base + deg[2 + i];
    cand_cnt[q] = n_odd;
}

__global__ void fill_i32_kernel(int *p, int v, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
// Fallback selection: a query whose candidate list overflowed, or whose own norm is degenerate, is re-done by the exact
// scan.  qsel[0] = number of selected queries, qsel[1..] their indices.  flags[0] = that number (stats), flags[3] counts
// searches that needed any fallback.
__global__ void select_fallback_kernel(const uint32_t *__restrict__ cnt, uint32_t cap, const float *__restrict__ qmags,
                                       uint32_t n, uint32_t *qsel, uint32_t *flags) {
    __shared__ uint32_t total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const bool bad = cnt[i] > cap || (qmags && !norm_is_proper(qmags[i]));
        if (bad) qsel[1 + atomicAdd(&total, 1u)] = i;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        qsel[0] = total;
        flags[0] = total;
        if (total) flags[3] += 1;
    }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

cdb_status make_tensor_map_2d(CUtensorMap *map, CUtensorMapDataType dtype, uint32_t elem_bytes, const void *base, uint64_t rows,
                              uint32_t cols, uint64_t pitch_bytes, uint32_t box_rows) {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        CDB_CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        if (!p || q != cudaDriverEntryPointSuccess) { set_error("cuTensorMapEncodeTiled not available"); return CDB_CUDA_ERROR; }
        fn = (PFN_encodeTiled)p;
    }
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {(cuuint64_t)pitch_bytes};
    cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, dtype, 2, const_cast<void *>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed: " + std::to_string((int)r)); return CDB_CUDA_ERROR; }
    return CDB_OK;
}
static cdb_status make_map_f16(CUtensorMap *map, const void *base, uint64_t rows, uint32_t dim, uint32_t pitch_halfs, uint32_t box_rows) {
    return make_tensor_map_2d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, rows, dim, (uint64_t)pitch_halfs * 2, box_rows);
}

static int tensor_scan_stages(uint32_t k) {
    if (k > (uint32_t)TS_GROUPS) return 0;  // the class-maximum bound needs k <= 64 disjoint classes
    return TS_STAGES;
}
static size_t tensor_scan_smem(int stages) {
    // tiles + candidate staging + barriers + (integer form) reciprocal magnitudes of two tiles + flags
    return 1024 + (size_t)stages * TS_STAGE_BYTES + (size_t)TS_CONSUMERS * 2 * TS_STAGE_SLOT_BYTES + 2 * stages * 8 +
           2 * TS_BLOCK_N * 4 + 16;
}
size_t tensor_scan_smem_bytes(uint32_t k) {
    if (!tensor_scan_stages(k)) return (size_t)1 << 30;
    return tensor_scan_smem(TS_STAGES);
}

template <int NG, bool HAS_DEG, int KIND>
static cdb_status launch_tensor_scan_gd(const CUtensorMap &mq, const CUtensorMap &mx, const TensorScanArgs &a, uint32_t grid,
                                        cudaStream_t s) {
    auto kern = tensor_scan_kernel<TS_STAGES, NG, HAS_DEG, KIND>;
    const size_t smem = tensor_scan_smem(TS_STAGES);
    CDB_ALLOW_SMEM(kern, smem);
    kern<<<grid, TS_THREADS, smem, s>>>(mq, mx, a);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

template <int NG, int KIND>
static cdb_status launch_tensor_scan_g(const CUtensorMap &mq, const CUtensorMap &mx, const TensorScanArgs &a, uint32_t grid, cudaStream_t s) {
    if (KIND == 1) return launch_tensor_scan_gd<NG, false, KIND>(mq, mx, a, grid, s);   // exact scores: no degenerate-row variant
    return a.has_deg ? launch_tensor_scan_gd<NG, true, 0>(mq, mx, a, grid, s)
                     : launch_tensor_scan_gd<NG, false, 0>(mq, mx, a, grid, s);
}

// fewer classes = cheaper bound refresh (the sort network grows as NG log^2 NG); the bound stays within ~1.5x of the
// exact k-th best as long as k is well below NG
template <int KIND>
static cdb_status launch_tensor_scan(const CUtensorMap &mq, const CUtensorMap &mx, const TensorScanArgs &a, uint32_t grid, cudaStream_t s) {
    if (a.k <= 12) return launch_tensor_scan_g<16, KIND>(mq, mx, a, grid, s);
    if (a.k <= 28) return launch_tensor_scan_g<32, KIND>(mq, mx, a, grid, s);
    return launch_tensor_scan_g<64, KIND>(mq, mx, a, grid, s);
}

// seeding pass over a prefix of the corpus, then the main pass (both forms)
template <int KIND>
static cdb_status run_tensor_scan(const CUtensorMap &mq, const CUtensorMap &mx, TensorScanArgs a, uint64_t n_rows,
                                  uint32_t *d_progress, int sm_count, cudaStream_t s) {
    cdb_status rc;
    // 1. seeding pass over a prefix of the corpus: a few CTAs per query tile, no emission, only the class maxima.
    //    Afterwards every CTA of the main pass starts from the k-th best of ~16K rows instead of from
    //    -inf, which removes the per-CTA warm-up bursts from the candidate lists.
    const uint32_t seed_tiles = std::min<uint32_t>(a.ntiles, 64);
    a.progress = d_progress;
    if (a.ntiles > 8) {
        TensorScanArgs sa = a;
        sa.emit = 0;
        sa.ntiles = seed_tiles;
        sa.n_rows = std::min<uint64_t>(n_rows, (uint64_t)seed_tiles * TS_BLOCK_N);
        // as many CTAs per query tile as the SMs allow, >= 2 corpus tiles each: the pass is a latency-bound prologue
        uint32_t per_m = std::max<uint32_t>(1, (uint32_t)sm_count / a.mtiles);
        per_m = std::min<uint32_t>(per_m, std::max<uint32_t>(1, seed_tiles / 2));
        const uint32_t sgrid = a.mtiles * per_m;
        if ((rc = launch_tensor_scan<KIND>(mq, mx, sa, sgrid, s))) return rc;
    }
    // 2. main pass.  Every CTA should own several corpus tiles, so tiny corpora are not shredded over all SMs.
    a.emit = 1;
    uint64_t total_tiles = (uint64_t)a.mtiles * a.ntiles;
    uint32_t grid = (uint32_t)std::min<uint64_t>((uint64_t)sm_count, std::max<uint64_t>(1, total_tiles / 4));
    grid = std::max<uint32_t>(1, grid / a.mtiles) * a.mtiles;  // whole groups only (132 SMs, 16 query tiles -> 128 CTAs)
    if (grid > (uint32_t)sm_count) { set_error("tensor scan: more query tiles than SMs"); return CDB_INVALID_PARAMS; }
    a.progress = d_progress + 1024;   // the seeding pass used the first 1024 counters
    return launch_tensor_scan<KIND>(mq, mx, a, grid, s);
}

// d_xh: fp16 normalised corpus [n_rows][pitch_halfs]; d_qh: fp16 normalised queries, padded with zero
// rows to a multiple of 128 [mtiles*128][pitch_halfs].
cdb_status tensor_scan_device(const void *d_xh, const void *d_qh, uint32_t pitch_halfs, uint64_t n_rows, uint32_t nq,
                              uint32_t dim, uint32_t k, float two_eps, uint32_t id_base, int *d_ggm, uint32_t *d_cand,
                              uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_progress, const uint32_t *d_deg, bool has_deg,
                              int sm_count, cudaStream_t s, bool prepared) {
    TensorScanArgs a{};
    a.has_deg = has_deg ? 1u : 0u;
    a.progress = d_progress;
    a.window = 3;
    a.refresh_mask = 15;
    if (const char *e = getenv("CDB_TS_WINDOW")) a.window = (uint32_t)atoi(e);      // tuning knobs (bench experiments)
    if (const char *e = getenv("CDB_TS_REFRESH")) a.refresh_mask = (uint32_t)atoi(e);
    a.n_rows = n_rows;
    a.n_queries = nq;
    a.k = k;
    a.kblocks = (dim + TS_BLOCK_K - 1) / TS_BLOCK_K;
    a.mtiles = (nq + TS_BLOCK_M - 1) / TS_BLOCK_M;
    a.ntiles = (uint32_t)((n_rows + TS_BLOCK_N - 1) / TS_BLOCK_N);
    a.two_eps = two_eps;
    a.id_base = id_base;
    a.ggm = d_ggm;
    a.cand = d_cand;
    a.cand_cnt = d_cand_cnt;
    a.cand_cap = cand_cap;
    const int stages = tensor_scan_stages(k);
    if (!stages) { set_error("tensor scan: k too large for shared memory"); return CDB_INVALID_PARAMS; }
    CUtensorMap mq, mx;
    cdb_status rc;
    if ((rc = make_map_f16(&mq, d_qh, (uint64_t)a.mtiles * TS_BLOCK_M, dim, pitch_halfs, TS_BLOCK_M))) return rc;
    if ((rc = make_map_f16(&mx, d_xh, n_rows, dim, pitch_halfs, TS_BLOCK_N))) return rc;
    if (!prepared) {   // prep_queries_kernel did all of this already
        fill_i32_kernel<<<(a.mtiles * TS_BLOCK_M * TS_GROUPS + 255) / 256, 256, 0, s>>>(d_ggm, (int)0x807FFFFF /* f2ord(-inf) */, a.mtiles * TS_BLOCK_M * TS_GROUPS);
        CDB_LAUNCH_CHECK();
        if (has_deg) {
            seed_candidates_kernel<<<(nq + 255) / 256, 256, 0, s>>>(d_deg, id_base, nq, d_cand, cand_cap, d_cand_cnt);
            CDB_LAUNCH_CHECK();
        } else {
            CDB_CUDA_TRY(cudaMemsetAsync(d_cand_cnt, 0, (size_t)nq * 4, s));
        }
        CDB_CUDA_TRY(cudaMemsetAsync(d_progress, 0, 8192, s));
    }

    a.rel = 1.0f;
    return run_tensor_scan<0>(mq, mx, a, n_rows, d_progress, sm_count, s);
}

// Integer form (tensor_scan_u8.cu): d_x u8 operand rows [n_rows][pitch] (u8 codes or unpacked digits), d_q the query operand
// rows padded with zero rows to a multiple of 128.  Emits exact selection keys into d_cand64; the caller sorts them.
cdb_status tensor_scan_i8_device(const uint8_t *d_x, const uint8_t *d_q, uint32_t pitch, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, int metric, const float *d_mags, const float *d_qmags, uint32_t id_base, int *d_ggm,
                                 uint64_t *d_cand64, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_err32, uint32_t *d_progress,
                                 int sm_count, cudaStream_t s) {
    TensorScanArgs a{};
    a.window = 3;
    a.refresh_mask = 15;
    a.n_rows = n_rows;
    a.n_queries = nq;
    a.k = k;
    a.kblocks = (dim + 2 * TS_BLOCK_K - 1) / (2 * TS_BLOCK_K);   // 128 u8 elements per 128-byte row
    a.mtiles = (nq + TS_BLOCK_M - 1) / TS_BLOCK_M;
    a.ntiles = (uint32_t)((n_rows + TS_BLOCK_N - 1) / TS_BLOCK_N);
    a.two_eps = 0.0f;
    a.rel = metric == CDB_METRIC_COSINE ? 1.0f - 1.0f / 262144.0f : 1.0f;
    a.id_base = id_base;
    a.ggm = d_ggm;
    a.cand64 = d_cand64;
    a.cand_cnt = d_cand_cnt;
    a.cand_cap = cand_cap;
    a.metric = metric;
    a.mags = d_mags;
    a.qmags = d_qmags;
    a.err32 = d_err32;
    if (!tensor_scan_stages(k)) { set_error("u8 tensor scan: k too large (class-maximum bound needs k <= 64)"); return CDB_INVALID_PARAMS; }
    if ((uint32_t)sm_count < a.mtiles) { set_error("u8 tensor scan: more query tiles than SMs"); return CDB_INVALID_PARAMS; }
    CUtensorMap mq, mx;
    cdb_status rc;
    if ((rc = make_tensor_map_2d(&mq, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, d_q, (uint64_t)a.mtiles * TS_BLOCK_M, dim, pitch, TS_BLOCK_M))) return rc;
    if ((rc = make_tensor_map_2d(&mx, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, d_x, n_rows, dim, pitch, TS_BLOCK_N))) return rc;
    fill_i32_kernel<<<(a.mtiles * TS_BLOCK_M * TS_GROUPS + 255) / 256, 256, 0, s>>>(d_ggm, (int)0x807FFFFF /* f2ord(-inf) */, a.mtiles * TS_BLOCK_M * TS_GROUPS);
    CDB_LAUNCH_CHECK();
    CDB_CUDA_TRY(cudaMemsetAsync(d_cand_cnt, 0, (size_t)nq * 4, s));
    CDB_CUDA_TRY(cudaMemsetAsync(d_progress, 0, 8192, s));
    return run_tensor_scan<1>(mq, mx, a, n_rows, d_progress, sm_count, s);
}

cdb_status select_fallback_device(const uint32_t *d_cnt, uint32_t cap, const float *d_qmags, uint32_t n, uint32_t *d_qsel,
                                  uint32_t *d_flags, cudaStream_t s) {
    select_fallback_kernel<<<1, 1024, 0, s>>>(d_cnt, cap, d_qmags, n, d_qsel, d_flags);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // namespace cdb
