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
// arithmetic, so the final ids/scores are bit-identical to the exact scan (the s8 form first drops the candidates that
// fail its filter against the final bound, s8_refilter_kernel).
//
// Kernel anatomy (one CTA per SM, 384 threads):
//   warps 0..7   two consumer warpgroups: wgmma M64 x N256 x K16 on their half of the query tile, accumulators in
//                registers, then the threshold epilogue straight from those registers (setmaxnreg: 232 registers)
//   warps 8..11  producer warpgroup (setmaxnreg: 40 registers), one thread issues the TMA loads:
//                cp.async.bulk.tensor.2d, SWIZZLE_128B, 4-stage mbarrier ring
// Tile: 128 queries (A, K-major) x 256 corpus rows (B, K-major), K block = 64 halfs (128 B).
// The s8 form at k <= 12 and D <= 1024 runs tensor_scan_s8_kernel instead: query tile resident, the two consumer
// warpgroups on the two 128-row halves of each corpus tile, taking turns at the tensor pipe.
#include <atomic>
#include <climits>
#include <cmath>
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
// clock64 sums of the instrumented instantiation (PROF): consumer slots summed over both warpgroups (thread 0 of each),
// producer slots over the issuing thread, all over every CTA of every launch since the sums were last read
enum : int {
    TS_PROF_FULL_WAIT,   // consumers waiting on a full barrier (starved of operands)
    TS_PROF_MMA,         // consumers issuing the k-blocks' wgmma and waiting for them to retire
    TS_PROF_EPILOGUE,    // class maxima, threshold test, emission (and the KIND 1 cosine staging) up to the bound refresh
    TS_PROF_REFRESH,     // the bound refresh
    TS_PROF_EMPTY_WAIT,  // producer waiting on an empty barrier (ring full)
    TS_PROF_DRIFT,       // producer in the bounded-drift spin
    TS_PROF_TILES,       // tiles processed (per warpgroup)
    TS_PROF_CONSUMER,    // consumers: whole tile loop
    TS_PROF_PRODUCER,    // producer: whole issue loop
    TS_PROF_CTAS,        // CTAs
    TS_PROF_MATH_WAIT,   // s8 form: consumers waiting for their turn at the tensor pipe (the other warpgroup's K loop)
    TS_PROF_EPI_THR,     // s8 form, parts of TS_PROF_EPILOGUE: the four queries' thresholds (while the turn's MMAs drain)
    TS_PROF_EPI_FOLD,    //   the per-class fold into gm and the shared class maxima (only where a class can grow)
    TS_PROF_EPI_EMIT,    //   the emission loops (only on a hit)
    TS_PROF_BOUND_ROUNDS,   // s8 form: rounds of the bound warp (TS_PROF_REFRESH then sums the bound warp's clocks in them)
    TS_PROF_EPI_CMAX,    // s8 form, part of TS_PROF_EPILOGUE: class maxima, hit test and the test whether a class can grow
    TS_PROF_SLOTS
};

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
    uint32_t refresh_mask;  // tensor_scan_kernel: the shared bound is refreshed when (tile & mask) == mask (and for the
                            // first tiles); tensor_scan_s8_kernel refreshes it in its bound warp instead
    uint32_t has_deg;       // the corpus holds degenerate rows: kernel variant that keeps zero accumulators out of the bound
    unsigned long long *prof;   // [TS_PROF_SLOTS] clock64 sums of the instrumented instantiation, null otherwise
    // ---- integer form (KIND 1: exact scoring of u8 codes / sub-byte digits on wgmma .s32.u8.u8, tensor_scan_u8.cu)
    int metric;             // CDB_METRIC_COSINE or CDB_METRIC_DOT_PRODUCT
    const float *mags;      // [n_rows] stored magnitudes (cosine)
    const float *qmags;     // [n_queries]
    uint64_t *cand64;       // [n_queries][cand_cap] emitted selection keys (exact scores)
    uint32_t *err32;        // [n_queries] error bits
    float rel;              // threshold = bound * rel - two_eps (1 for the f16 form and for the dot product; 1 - 2^-18 for cosine)
    const uint32_t *deleted;   // deleted-row bitmap (bit r = row r), null while no row is deleted: a corpus tile is 8 words
    // ---- s8 form (KIND 2: the prefilter on wgmma .s32.s8.s8 against the s8 shadow, DESIGN.md section 5c)
    const float2 *tile_se;  // [ntiles] {s_T, E_T} of each corpus tile
    const float2 *q_se;     // [n_queries] {s_q, e_q}
    const float2 *tile_rcp; // [ntiles] {1/s_T rounded down, rounded up} (tensor_scan_s8_kernel)
    const float2 *q_rcp;    // [n_queries] {1/s_q rounded down, rounded up} (tensor_scan_s8_kernel)
    float dn1;              // 1 + delta_n, rounded up: bound on |x_hat| and |q_hat|
    float dref;             // delta_ref(D), rounded up: the reference's f32 cosine against the exact q_hat . x_hat
    uint32_t stages;        // tensor_scan_s8_kernel: depth of its corpus ring (16 KB stages)
};

// Candidate staging in shared memory: 40 bytes per (consumer thread, query row): slot 0 = count, then 9 row ids (f16 form)
// resp. 4 selection keys (integer form)
constexpr uint32_t TS_STAGE_SLOT_BYTES = 40;
constexpr uint32_t TS_LSTAGE = 9;
constexpr uint32_t TS_KSTAGE = 4;
constexpr int TS_GROUPS = 64;       // at most 64 class maxima per query; the filter supports k <= TS_GROUPS

// bit r of a row bitmap (null: no bit is set)
__device__ __forceinline__ bool bit_is_set(const uint32_t *bits, uint64_t r) { return bits && ((bits[r >> 5] >> (r & 31)) & 1u); }

// rare path: one approximate score passed the threshold -> stage the row id, flush CAP at a time
// (the few fields it needs by value: a reference to the kernel's arguments would copy them to the stack)
template <uint32_t CAP = TS_LSTAGE>
__device__ __noinline__ void epi_emit(uint32_t *cand, uint32_t *cand_cnt, uint32_t cand_cap, uint32_t qi, uint32_t *stage, uint32_t id) {
    uint32_t c = stage[0];
    stage[1 + c] = id;
    if (++c == CAP) {
        const uint32_t pos = atomicAdd(cand_cnt + qi, c);
        for (uint32_t i = 0; i < c; ++i)
            if (pos + i < cand_cap) cand[(size_t)qi * cand_cap + pos + i] = stage[1 + i];
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

// word x (0..7) of the deleted-row bitmap over the corpus tile starting at row0 (rows past the corpus: 0)
__device__ __forceinline__ uint32_t tile_word(const TensorScanArgs &a, uint64_t row0, int x) {
    return row0 + 32 * x < a.n_rows ? __ldg(a.deleted + (row0 >> 5) + x) : 0u;
}
// the deleted bits of a consumer thread's 64 columns 8j + 2qd + b, as bit 2j + b
__device__ __forceinline__ uint64_t tile_dead(const TensorScanArgs &a, uint64_t row0, uint32_t qd) {
    uint64_t dead = 0;
#pragma unroll
    for (int x = 0; x < 8; ++x) {
        const uint32_t sw = tile_word(a, row0, x) >> (2 * qd);   // bits 8m + {0,1}: columns 32x + 8m + 2qd + {0,1}
        dead |= (uint64_t)((sw & 0x3u) | ((sw >> 6) & 0xCu) | ((sw >> 12) & 0x30u) | ((sw >> 18) & 0xC0u)) << (8 * x);
    }
    return dead;
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
// KIND = 2: the prefilter of KIND 0 on wgmma .s32.s8.s8 (twice the f16 rate, half the operand bytes): s8 codes of the
// normalised rows / queries with one scale per corpus tile (s_T) and per query (s_q), 128 bytes of K per stage like KIND 1.
// An s32 accumulator dp scores s_T*s_q*dp with |s_T*s_q*dp - cos_ref| <= eps(q,T) (DESIGN.md section 5c).  Per value the
// epilogue keeps integer class maxima; once per tile and query it folds their rigorous lower bounds
// fl_down(cm*s_T*s_q) - eps(q,T) into the float class maxima and turns the threshold A into the integer
// thrI = floor((A - eps(q,T)) / (s_T*s_q)) (directed rounding throughout): a row is emitted iff dp >= thrI, i.e. iff its
// upper bound reaches A.
//
// Register layout of the epilogue: a consumer thread holds two query rows (r and r + 8 of its warpgroup's 64) and, of each,
// the 64 columns 8j + 2(lane%4) + {0,1}.  Classes are column mod NG, so the thread owns NG/4 classes of each of its queries
// (those = 2(lane%4) or 2(lane%4)+1 mod 8); the four threads of a quad together cover all NG classes of their two queries.
//
// PROF: the instrumented instantiation (a.prof): clock64 sums per phase, see TS_PROF_*.
template <int STAGES, int NG, bool HAS_DEG, int KIND, bool PROF>
__global__ void __launch_bounds__(TS_THREADS, 1)
tensor_scan_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_x, TensorScanArgs a) {
    constexpr uint32_t K_ELEMS = KIND != 0 ? 2 * TS_BLOCK_K : TS_BLOCK_K;   // elements per 128-byte row: 128 u8/s8 / 64 halfs
    constexpr int NL = NG / 4;                                              // classes a thread owns per query
    using Acc = typename std::conditional<KIND != 0, uint32_t, float>::type;
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
            unsigned long long p_empty = 0, p_drift = 0, p_t0 = PROF ? clock64() : 0;
            uint32_t s = 0, phase = 0, t = 0;
            for (uint32_t nt = g; nt < a.ntiles; nt += G, ++t) {
                if (a.mtiles > 1 && t >= a.window) {
                    const unsigned long long c0 = PROF ? clock64() : 0;
                    // bounded drift: every CTA of the group must have consumed tile t - window
                    const uint32_t need = (t - a.window + 1) * a.mtiles;
                    // bounded spin: if a peer CTA is not resident (GPU shared with another stream) we only lose locality
                    for (int spin = 0; spin < 20000 && *reinterpret_cast<volatile uint32_t *>(a.progress + g) < need; ++spin) __nanosleep(64);
                    if (PROF) p_drift += clock64() - c0;
                }
                for (uint32_t kb = 0; kb < a.kblocks; ++kb) {
                    const unsigned long long c0 = PROF ? clock64() : 0;
                    mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
                    if (PROF) p_empty += clock64() - c0;
                    const uint32_t fb = smem_u32(&full_bar[s]);
                    const uint32_t sa = smem_u32(tiles + (size_t)s * TS_STAGE_BYTES);
                    mbar_expect_tx(fb, TS_STAGE_BYTES);
                    tma_load_2d(sa, &map_q, fb, (int)(kb * K_ELEMS), (int)(mt * TS_BLOCK_M));
                    tma_load_2d(sa + TS_A_BYTES, &map_x, fb, (int)(kb * K_ELEMS), (int)(nt * TS_BLOCK_N));
                    if (++s == STAGES) { s = 0; phase ^= 1; }
                }
            }
            if (PROF) {
                atomicAdd(a.prof + TS_PROF_EMPTY_WAIT, p_empty);
                atomicAdd(a.prof + TS_PROF_DRIFT, p_drift);
                atomicAdd(a.prof + TS_PROF_PRODUCER, clock64() - p_t0);
                atomicAdd(a.prof + TS_PROF_CTAS, 1ull);
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
        float2 qse[2];   // KIND 2: {s_q, e_q}
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const uint32_t ql = qrow0 + 8 * i;
            qi[i] = mt * TS_BLOCK_M + ql;
            qvalid[i] = qi[i] < a.n_queries;
            qmag[i] = (KIND == 1 && qvalid[i]) ? a.qmags[qi[i]] : 0.0f;
            if (KIND == 2) qse[i] = qvalid[i] ? a.q_se[qi[i]] : make_float2(0.0f, 0.0f);
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
        unsigned long long p_full = 0, p_mma = 0, p_epi = 0, p_ref = 0, p_c = PROF ? clock64() : 0;
        uint32_t s = 0, phase = 0, t = 0;
        for (uint32_t nt = g; nt < a.ntiles; nt += G, ++t) {
            const uint64_t row0 = (uint64_t)nt * TS_BLOCK_N;
            const float *rs = rinv_s + (t & 1) * TS_BLOCK_N;
            unsigned long long c_tile = PROF ? clock64() : 0, c_full = 0;
            // KIND 2: {s_T, E_T}, loaded before the MMAs so that its L2 round trip hides under them
            const float2 se = KIND == 2 ? __ldg(a.tile_se + nt) : make_float2(0.0f, 0.0f);
            if (cosine) {
                // reciprocal magnitudes of this tile's rows -> shared memory (double buffered by tile parity); a zero
                // magnitude is an Err for every query that meets the row (cosine.rs:230-231)
                if (ct == 0) zflag_s[t & 1] = 0u;
                asm volatile("bar.sync 1, 256;" ::: "memory");
                const bool valid = row0 + ct < a.n_rows;
                const float mg = valid ? a.mags[row0 + ct] : 0.0f;
                rinv_s[(t & 1) * TS_BLOCK_N + ct] = mg > 0.0f ? __frcp_rn(mg) : 0.0f;
                // a deleted row raises no Err (as in the exact scan)
                if (valid && mg == 0.0f && !bit_is_set(a.deleted, row0 + ct)) zflag_s[t & 1] = 1u;
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (zflag_s[t & 1]) {
#pragma unroll
                    for (int i = 0; i < 2; ++i) if (qvalid[i]) err[i] |= (uint32_t)CDB_ERRFLAG_CALCULATION;
                }
            }
            // ---- the tile's product: kblocks x 4 wgmma into registers; a stage is released when its MMAs have retired.
            //      The zeroing costs 128 moves per thread and tile, but it is what ends the accumulators' live range for
            //      ptxas: a wgmma with scale-d 0 still reads them, so without it they stay live through the epilogue and
            //      the NG = 64 instantiations spill.
            const unsigned long long c_main = PROF ? clock64() : 0;
            Acc acc[128];
#pragma unroll
            for (int i = 0; i < 128; ++i) acc[i] = 0;
            uint32_t prev = 0;
            for (uint32_t kb = 0; kb < a.kblocks; ++kb) {
                const unsigned long long c0 = PROF ? clock64() : 0;
                mbar_wait(smem_u32(&full_bar[s]), phase);
                if (PROF) c_full += clock64() - c0;
                const uint32_t sa = sa0 + s * TS_STAGE_BYTES;
                const uint64_t adesc = make_smem_desc(sa + wg * (TS_A_BYTES / 2)), bdesc = make_smem_desc(sa + TS_A_BYTES);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {  // +32 bytes along K = +2 in the encoded start address
                    if constexpr (KIND == 1) wgmma_u8(acc, adesc + 2 * kk, bdesc + 2 * kk);
                    else if constexpr (KIND == 2) wgmma_s8(acc, adesc + 2 * kk, bdesc + 2 * kk);
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
            unsigned long long c_epi = 0;
            if (PROF) {
                c_epi = clock64();
                p_full += c_full;
                p_mma += c_epi - c_main - c_full;
                p_epi += c_main - c_tile;   // KIND 1 cosine: the per-tile reciprocal staging
            }

            // ---- epilogue: fold the values into the class maxima, test the tile maximum against the threshold,
            //      build the per-value tests only on a hit
            // KIND 1 (its operands are the stored codes, so deleted rows cannot be zeroed like the shadows of KIND 0 / 2):
            // every thread reads the tile's 8 bitmap words, so `dirty` is uniform; a dirty tile takes the masked epilogue
            bool dirty = false;
            if constexpr (KIND == 1) {
                if (a.deleted) {
#pragma unroll
                    for (int x = 0; x < 8; ++x) dirty |= tile_word(a, row0, x) != 0u;
                }
            }
            const uint64_t dead = dirty ? tile_dead(a, row0, qd) : 0ull;   // bit 2j+b: column 8j + 2qd + b is a deleted row
            const bool full_tile = row0 + TS_BLOCK_N <= a.n_rows;   // only the corpus' last tile can be partial (TMA zero fill)
            const uint64_t left = a.n_rows > row0 ? a.n_rows - row0 : 0;   // valid columns of this tile
            if constexpr (KIND == 2) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    // s_T*s_q rounded down and up, eps(q,T) rounded up, thrI <= (A - eps) / (s_T*s_q)
                    const float slo = __fmul_rd(se.x, qse[i].x), shi = __fmul_ru(se.x, qse[i].x);
                    const float eps = __fmaf_ru(__fadd_ru(a.dn1, qse[i].y), se.y, __fmaf_ru(qse[i].y, a.dn1, a.dref));
                    const float num = __fsub_rd(bound[i], eps);
                    const int thrI = __float2int_rd(__fdiv_rd(num, num >= 0.0f ? shi : slo));
                    int cm[NL];
#pragma unroll
                    for (int l = 0; l < NL; ++l) cm[l] = INT_MIN;
                    bool hit;
                    if (full_tile) {
                        int zmax = INT_MIN;   // HAS_DEG: 0 if some accumulator of the tile is exactly zero
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
#pragma unroll
                            for (int b = 0; b < 2; ++b) {
                                int v = (int)acc[4 * j + 2 * i + b];
                                if (HAS_DEG) {
                                    zmax = v == 0 ? 0 : zmax;
                                    v = v == 0 ? INT_MIN : v;
                                }
                                const int l = (j & (NG / 8 - 1)) * 2 + b;
                                cm[l] = max(cm[l], v);
                            }
                        }
                        int cmax = zmax;
#pragma unroll
                        for (int l = 0; l < NL; ++l) cmax = max(cmax, cm[l]);
                        hit = cmax >= thrI;
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
#pragma unroll
                            for (int b = 0; b < 2; ++b) {
                                const uint32_t col = 8 * j + 2 * qd + b;
                                const int v = (int)acc[4 * j + 2 * i + b];
                                const int l = (j & (NG / 8 - 1)) * 2 + b;
                                if ((uint64_t)col < left && !(HAS_DEG && v == 0)) cm[l] = max(cm[l], v);
                            }
                        }
                        hit = true;
                    }
                    // |dp| < 2^31 (127^2 * D, D <= rerank_f32_max_dim()): INT_MIN only marks an empty class
#pragma unroll
                    for (int l = 0; l < NL; ++l)
                        if (cm[l] != INT_MIN)
                            gm[i][l] = fmaxf(gm[i][l], __fsub_rd(__fmul_rd(__int2float_rd(cm[l]), cm[l] >= 0 ? slo : shi), eps));
                    if (qvalid[i] && a.emit && hit) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
#pragma unroll
                            for (int b = 0; b < 2; ++b) {
                                const uint32_t col = 8 * j + 2 * qd + b;
                                if ((uint64_t)col < left && (int)acc[4 * j + 2 * i + b] >= thrI)
                                    epi_emit(a.cand, a.cand_cnt, a.cand_cap, qi[i], stage[i], a.id_base + (uint32_t)(row0 + col));
                            }
                        }
                    }
                }
            } else {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                bool hit;
                if (full_tile && !dirty) {
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
                } else {   // the corpus' partial last tile, or (KIND 1) a tile with deleted rows: they stay out of the bound
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
#pragma unroll
                        for (int b = 0; b < 2; ++b) {
                            const uint32_t col = 8 * j + 2 * qd + b;
                            const float v = acc_value<KIND>(acc[4 * j + 2 * i + b], cosine, cosine ? rs[col] : 0.0f);
                            const int l = (j & (NG / 8 - 1)) * 2 + b;
                            if ((uint64_t)col < left && !(HAS_DEG && v == 0.0f) && !((dead >> (2 * j + b)) & 1u))
                                gm[i][l] = fmaxf(gm[i][l], v);
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
                            if ((uint64_t)col < left && !((dead >> (2 * j + b)) & 1u) && v >= thr[i]) {
                                if (KIND == 1) epi_emit_key(a, qi[i], kstage[i], (int)acc_bits(acc[4 * j + 2 * i + b]), row0 + col, qmag[i]);
                                else epi_emit(a.cand, a.cand_cnt, a.cand_cap, qi[i], stage[i], a.id_base + (uint32_t)(row0 + col));
                            }
                        }
                    }
                }
            }
            }
            unsigned long long c_ref = 0;
            if (PROF) {
                c_ref = clock64();
                p_epi += c_ref - c_epi;
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
            if (PROF) p_ref += clock64() - c_ref;
        }
        if (PROF && (ct & 127) == 0) {
            atomicAdd(a.prof + TS_PROF_FULL_WAIT, p_full);
            atomicAdd(a.prof + TS_PROF_MMA, p_mma);
            atomicAdd(a.prof + TS_PROF_EPILOGUE, p_epi);
            atomicAdd(a.prof + TS_PROF_REFRESH, p_ref);
            atomicAdd(a.prof + TS_PROF_TILES, (unsigned long long)t);
            atomicAdd(a.prof + TS_PROF_CONSUMER, clock64() - p_c);
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

// ------------------------------------------------------------------ s8 form: ping-pong consumers, query tile resident
// tensor_scan_s8_kernel runs the KIND 2 filter of tensor_scan_kernel with the tile's work split differently, so that one
// warpgroup's epilogue runs while the other warpgroup's MMAs keep the tensor pipe busy:
//   * the CTA's 128 x D query tile is loaded once and stays in shared memory (the ring carries corpus rows only);
//   * warpgroup w takes rows [128w, 128w + 128) of every 256-row corpus tile: all 128 queries x 128 rows as two
//     m64n128k32 wgmma chains (queries 0-63 and 64-127), 128 s32 accumulators per thread as before;
//   * an ordered pair of named barriers hands the tensor pipe from one warpgroup's K loop to the other's
//     (0, 1, 0, 1, ...); each warpgroup takes exactly one turn per corpus tile of the CTA, a half past the corpus end
//     included (its stages arrive without data and its values are masked), so the turns always pair up;
//   * the ring is one sequence of 16 KB stages (128 rows x 128 B): tile t's lower half's k-blocks, then its upper half's.
//     Turns consume it in that order, so the producer only ever waits for a stage an earlier turn releases;
//   * the bound refresh runs in a warp of its own, the bound warp (warp 1 of the producer warpgroup): the consumers raise
//     the CTA's class maxima in shared memory (`cls`, shared atomicMax, only when a value grew) and read the queries'
//     bounds from `sbound`; they never touch the global class maxima during the scan.  A bound-warp round pushes the
//     CTA's class maxima that exceed the global ones to `ggm` (RED), takes the k-th largest of each query's NG class
//     maxima (the larger of the global and the CTA's value) by rank counting, and raises `sbound`.  It runs once per
//     warpgroup epilogue (woken as the epilogue starts; back to back when it falls behind).  It only moves and selects
//     values the consumers computed as rigorous lower bounds, and `sbound` only rises, so a stale bound costs
//     candidates, never correctness.
// Shared memory (227 KB per block): query tile kblocks x 16 KB (96 KB at D = 768) + ring stages x 16 KB (6: one whole
// half-tile at D = 768) + candidate staging 256 threads x 4 queries x 16 B (a count and 3 ids: 16 KB) + class maxima
// NG x 128 ints (8 KB) + per query the bound, {s_q, 1/s_q down, 1/s_q up, 1 + delta_n + e_q} and e_q (1 + delta_n) +
// delta_ref (3 KB) + control words + barriers.
// Register layout of the epilogue: a thread holds 4 query rows, 16 wl + lane/4 + {0, 8} + {0, 64}, and of each the 32
// columns 8j + 2(lane%4) + {0,1} of its warpgroup's half.  The half's offset (128) is a multiple of NG, so a column's class
// (column mod NG) is the same as in tensor_scan_kernel and each thread owns NG/4 classes of each of its queries.
constexpr uint32_t TS8_HALF = 128;                       // corpus rows per warpgroup turn
constexpr uint32_t TS8_KB_BYTES = 128 * 128;             // one k-block of the query tile or of a half-tile
constexpr uint32_t TS8_MAX_STAGES = 6;
constexpr uint32_t TS8_MIN_STAGES = 4;                   // fewer: the streamed kernel (tensor_scan_kernel) runs instead
constexpr uint32_t TS8_SLOT_BYTES = 16;
constexpr uint32_t TS8_LSTAGE = TS8_SLOT_BYTES / 4 - 1;  // ids staged per (thread, query)
constexpr int TS8_NG = 16;                               // the kernel runs k <= 12 (NG = 16) only
constexpr int TS8_BAR_TURN = 2;                          // named barriers 2 and 3: "warpgroup 0 / 1 may issue its K loop"
constexpr uint32_t TS8_BOUND_WARP = TS_CONSUMERS / 32 + 1;
constexpr size_t TS8_SMEM_FIXED = 1024 + (size_t)TS_CONSUMERS * 4 * TS8_SLOT_BYTES + (size_t)TS8_NG * TS_BLOCK_M * 4 +
                                  (size_t)TS_BLOCK_M * (4 + 16 + 4) + 16 + (2 * TS8_MAX_STAGES + 1) * 8;

// One bound-warp round over the CTA's query tile (lane: queries lane + 32j).  push: raise the global class maxima from the
// CTA's first.
template <int NG>
__device__ __forceinline__ void s8_bound_round(const TensorScanArgs &a, uint32_t mt, const int *cls, float *sbound, int lane, bool push) {
#pragma unroll 1
    for (int j = 0; j < TS_BLOCK_M / 32; ++j) {
        const uint32_t ql = lane + 32 * j;
        if (mt * TS_BLOCK_M + ql >= a.n_queries) break;
        int *gq = a.ggm + (size_t)mt * NG * TS_BLOCK_M + ql;
        int v[NG];
#pragma unroll
        for (int c = 0; c < NG; ++c) v[c] = *reinterpret_cast<const volatile int *>(gq + c * TS_BLOCK_M);
        if (push) {
#pragma unroll
            for (int c = 0; c < NG; ++c) {
                const int m = *reinterpret_cast<const volatile int *>(cls + c * TS_BLOCK_M + ql);
                if (m > v[c]) { atomicMax(gq + c * TS_BLOCK_M, m); v[c] = m; }
            }
        }
        // the k-th largest: the largest value that at least k of the NG values reach (ordered ints order like the floats)
        int b = INT_MIN;
#pragma unroll
        for (int i = 0; i < NG; ++i) {
            uint32_t n = 0;
#pragma unroll
            for (int c = 0; c < NG; ++c) n += v[c] >= v[i];
            b = n >= a.k ? max(b, v[i]) : b;
        }
        volatile float *sb = sbound + ql;
        if (ord2f(b) > *sb) *sb = ord2f(b);
    }
}

template <int NG, bool HAS_DEG, bool PROF>
__global__ void __launch_bounds__(TS_THREADS, 1)
tensor_scan_s8_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_x, TensorScanArgs a) {
    static_assert(NG <= TS8_NG, "the shared class maxima hold TS8_NG classes");
    constexpr int NL = NG / 4;   // classes a thread owns per query
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *qtile = smem;                                          // [kblocks] x 16 KB
    uint8_t *ring = qtile + (size_t)a.kblocks * TS8_KB_BYTES;       // [stages] x 16 KB
    uint8_t *lstage = ring + (size_t)a.stages * TS8_KB_BYTES;       // [256][4] x 16 B
    int *cls = reinterpret_cast<int *>(lstage + TS_CONSUMERS * 4 * TS8_SLOT_BYTES);   // [NG][128] CTA class maxima (ordered)
    float *sbound = reinterpret_cast<float *>(cls + TS8_NG * TS_BLOCK_M);             // [128] bound A of each query
    float4 *qpar = reinterpret_cast<float4 *>(sbound + TS_BLOCK_M);                   // [128] {s_q, 1/s_q down, up, eps_a}
    float *qeps = reinterpret_cast<float *>(qpar + TS_BLOCK_M);                       // [128] eps_b
    uint32_t *ctl = reinterpret_cast<uint32_t *>(qeps + TS_BLOCK_M);                  // [0] epilogues, [1] warpgroups done
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(ctl + 4);
    uint64_t *empty_bar = full_bar + TS8_MAX_STAGES, *q_bar = empty_bar + TS8_MAX_STAGES;

    const int lane = threadIdx.x & 31;
    const uint32_t mt = blockIdx.x % a.mtiles, g = blockIdx.x / a.mtiles, G = gridDim.x / a.mtiles;
    const uint32_t T = g < a.ntiles ? (a.ntiles - g + G - 1) / G : 0;   // corpus tiles g, g+G, ... of this CTA

    if (threadIdx.x == TS_CONSUMERS) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
        for (uint32_t s = 0; s < a.stages; ++s) { mbar_init(smem_u32(&full_bar[s]), 1); mbar_init(smem_u32(&empty_bar[s]), 4); }
        mbar_init(smem_u32(q_bar), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        ctl[0] = ctl[1] = 0;
    }
    for (uint32_t i = threadIdx.x; i < (uint32_t)NG * TS_BLOCK_M; i += TS_THREADS) cls[i] = (int)0x807FFFFF;   // f2ord(-inf)
    if (threadIdx.x < TS_BLOCK_M) {
        // per query: s_q and its reciprocals, and eps(q,T) = eps_a * E_T + eps_b rounded up (a padding row's values are
        // never used)
        const uint32_t qi = mt * TS_BLOCK_M + threadIdx.x;
        const float2 se = qi < a.n_queries ? a.q_se[qi] : make_float2(0.0f, 0.0f);
        const float2 rc = qi < a.n_queries ? a.q_rcp[qi] : make_float2(0.0f, 0.0f);
        qpar[threadIdx.x] = make_float4(se.x, rc.x, rc.y, __fadd_ru(a.dn1, se.y));
        qeps[threadIdx.x] = __fmaf_ru(se.y, a.dn1, a.dref);
        sbound[threadIdx.x] = -INFINITY;
    }
    __syncthreads();
    // what earlier launches (the seeding pass) and other CTAs already know, before the first epilogue reads it
    if (threadIdx.x / 32 == TS8_BOUND_WARP && T > 0) s8_bound_round<NG>(a, mt, cls, sbound, lane, false);
    __syncthreads();

    if (threadIdx.x >= TS_CONSUMERS) {
        // ===================== TMA producer and bound warp =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (threadIdx.x == TS_CONSUMERS && T > 0) {
            unsigned long long p_empty = 0, p_drift = 0, p_t0 = PROF ? clock64() : 0;
            mbar_expect_tx(smem_u32(q_bar), a.kblocks * TS8_KB_BYTES);
            for (uint32_t kb = 0; kb < a.kblocks; ++kb)
                tma_load_2d(smem_u32(qtile + (size_t)kb * TS8_KB_BYTES), &map_q, smem_u32(q_bar), (int)(kb * 128), (int)(mt * TS_BLOCK_M));
            uint32_t s = 0, phase = 0;
            for (uint32_t t = 0; t < T; ++t) {
                const uint32_t nt = g + t * G;
                if (a.mtiles > 1 && t >= a.window) {
                    const unsigned long long c0 = PROF ? clock64() : 0;
                    // bounded drift: every CTA of the group must have consumed tile t - window (as in tensor_scan_kernel)
                    const uint32_t need = (t - a.window + 1) * a.mtiles;
                    for (int spin = 0; spin < 20000 && *reinterpret_cast<volatile uint32_t *>(a.progress + g) < need; ++spin) __nanosleep(64);
                    if (PROF) p_drift += clock64() - c0;
                }
                for (uint32_t h = 0; h < 2; ++h) {
                    const uint64_t hrow0 = (uint64_t)nt * TS_BLOCK_N + h * TS8_HALF;
                    for (uint32_t kb = 0; kb < a.kblocks; ++kb) {
                        const unsigned long long c0 = PROF ? clock64() : 0;
                        mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
                        if (PROF) p_empty += clock64() - c0;
                        const uint32_t fb = smem_u32(&full_bar[s]);
                        if (hrow0 < a.n_rows) {
                            mbar_expect_tx(fb, TS8_KB_BYTES);
                            tma_load_2d(smem_u32(ring + (size_t)s * TS8_KB_BYTES), &map_x, fb, (int)(kb * 128), (int)hrow0);
                        } else {
                            mbar_arrive(fb);   // the upper half of a last tile that ends within its lower half: no rows
                        }
                        if (++s == a.stages) { s = 0; phase ^= 1; }
                    }
                }
            }
            if (PROF) {
                atomicAdd(a.prof + TS_PROF_EMPTY_WAIT, p_empty);
                atomicAdd(a.prof + TS_PROF_DRIFT, p_drift);
                atomicAdd(a.prof + TS_PROF_PRODUCER, clock64() - p_t0);
                atomicAdd(a.prof + TS_PROF_CTAS, 1ull);
            }
        } else if (threadIdx.x / 32 == TS8_BOUND_WARP && T > 0) {
            // one round per warpgroup epilogue, until the consumers have published their final class maxima
            unsigned long long p_ref = 0, n_rounds = 0;
            uint32_t seen = 0;
            for (;;) {
                uint32_t done, ep;
                for (;;) {
                    ep = __shfl_sync(0xffffffffu, *reinterpret_cast<volatile uint32_t *>(ctl), 0);
                    done = __shfl_sync(0xffffffffu, *reinterpret_cast<volatile uint32_t *>(ctl + 1), 0);
                    if (ep != seen || done == 2) break;
                    __nanosleep(128);
                }
                if (done == 2) break;
                seen = ep;
                const unsigned long long c0 = PROF ? clock64() : 0;
                s8_bound_round<NG>(a, mt, cls, sbound, lane, true);
                __syncwarp();
                if (PROF) { p_ref += clock64() - c0; ++n_rounds; }
            }
            if (PROF && lane == 0) {
                atomicAdd(a.prof + TS_PROF_REFRESH, p_ref);
                atomicAdd(a.prof + TS_PROF_BOUND_ROUNDS, n_rounds);
            }
        }
        return;
    }

    // ===================== consumers: MMA + threshold filter =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const uint32_t ct = threadIdx.x, wg = ct >> 7, wl = (ct >> 5) & 3, qd = (uint32_t)lane & 3;
    float gm[4][NL];   // this thread's share of the CTA's class maxima (the shared `cls` is raised whenever one grows)
    float gmin[4];     // min_l gm[i][l]: a tile whose largest lower bound does not exceed it raises none of them
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        reinterpret_cast<uint32_t *>(lstage + (size_t)(ct * 4 + i) * TS8_SLOT_BYTES)[0] = 0;
#pragma unroll
        for (int l = 0; l < NL; ++l) gm[i][l] = -INFINITY;
        gmin[i] = -INFINITY;
    }
    if (T == 0) return;
    if (wg == 1) named_bar_arrive<TS8_BAR_TURN, 256>();   // warpgroup 0 takes the first turn
    mbar_wait(smem_u32(q_bar), 0);
    const uint32_t q0 = smem_u32(qtile), r0 = smem_u32(ring);
    unsigned long long p_turn = 0, p_full = 0, p_mma = 0, p_thr = 0, p_cmax = 0, p_fold = 0, p_emit = 0, p_c = PROF ? clock64() : 0;
    for (uint32_t t = 0; t < T; ++t) {
        const uint32_t nt = g + t * G;
        const uint64_t row0 = (uint64_t)nt * TS_BLOCK_N + wg * TS8_HALF;   // this warpgroup's half
        // {s_T, E_T} and {1/s_T down, up} of the 256-row tile (both halves), loaded before the MMAs
        const float2 se = __ldg(a.tile_se + nt), rt = __ldg(a.tile_rcp + nt);
        // ring position of this turn's first k-block: turn 2t + wg of the sequence
        const uint32_t p0 = (2 * t + wg) * a.kblocks;
        uint32_t s = p0 % a.stages, phase = (p0 / a.stages) & 1u;
        unsigned long long c_turn = PROF ? clock64() : 0, c_full = 0;
        if (wg == 0) named_bar_sync<TS8_BAR_TURN, 256>();
        else named_bar_sync<TS8_BAR_TURN + 1, 256>();
        const unsigned long long c_main = PROF ? clock64() : 0;
        // the turn's first k-block overwrites the accumulators (scale-d 0) instead of 128 zeroing moves per turn
        uint32_t acc[128];
        uint32_t prev = 0;
        for (uint32_t kb = 0; kb < a.kblocks; ++kb) {
            const unsigned long long c0 = PROF ? clock64() : 0;
            mbar_wait(smem_u32(&full_bar[s]), phase);
            if (PROF) c_full += clock64() - c0;
            const uint32_t qa = q0 + kb * TS8_KB_BYTES;
            const uint64_t adesc0 = make_smem_desc(qa), adesc1 = make_smem_desc(qa + TS8_KB_BYTES / 2);
            const uint64_t bdesc = make_smem_desc(r0 + s * TS8_KB_BYTES);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {   // +32 bytes along K = +2 in the encoded start address
                wgmma_s8_n128(acc, adesc0 + 2 * kk, bdesc + 2 * kk, kb | kk);
                wgmma_s8_n128(acc + 64, adesc1 + 2 * kk, bdesc + 2 * kk, kb | kk);
            }
            wgmma_commit();
            wgmma_wait<1>();   // the previous k-block's MMAs have retired
            if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
            prev = s;
            if (++s == a.stages) { s = 0; phase ^= 1; }
        }
        // every MMA of the turn is issued: the other warpgroup may start its K loop while these drain.  Warpgroup 1's
        // last turn hands over nothing (warpgroup 0 has no turn left), so both barriers see as many arrivals as waits.
        if (wg == 0) named_bar_arrive<TS8_BAR_TURN + 1, 256>();
        else if (t + 1 < T) named_bar_arrive<TS8_BAR_TURN, 256>();
        const unsigned long long c_thr = PROF ? clock64() : 0;

        // ---- epilogue (the filter of tensor_scan_kernel, KIND 2).  Up to wgmma_wait<0> it needs no accumulator, so it
        //      runs while the turn's last MMAs drain.  The per-query addresses below are derived from `me`, which the empty
        //      asm makes opaque per tile: otherwise they are hoisted out of the tile loop and held in registers (or spilled)
        //      across the K loop, where the accumulators need every register.
        uint32_t me = ct;
        asm volatile("" : "+r"(me));
        // non-returning reductions that nothing below waits for.  progress: the tile's upper half is in (its K loop waited
        // for every one of its loads).  ctl: wakes the bound warp, which runs its rounds back to back at this cadence anyway.
        if (me == 128 && a.mtiles > 1) atomicAdd(a.progress + g, 1u);
        if ((me & 127) == 0) red_shared_add_u32(smem_u32(ctl), 1u);
        const uint32_t qrow = 16 * ((me >> 5) & 3) + ((me & 31) >> 2);   // + 8 (i & 1) + 64 (i >> 1)
        // the four queries' thresholds, as four independent chains.  s_T*s_q rounded down and up, eps(q,T) rounded up, and
        // thrI <= (A - eps) / (s_T*s_q) through the reciprocals rounded the safe way for the numerator's sign:
        // fl_down(fl_down(num * 1/s_T) * 1/s_q), down for num >= 0, up otherwise (s_T or s_q = 0: as the division did)
        float slo[4], shi[4], eps[4];
        int thrI[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t ql = qrow + 64 * (i >> 1) + 8 * (i & 1);
            const float4 qp = lds_f32x4(smem_u32(qpar + ql));
            slo[i] = __fmul_rd(se.x, qp.x);
            shi[i] = __fmul_ru(se.x, qp.x);
            eps[i] = __fmaf_ru(qp.w, se.y, lds_f32(smem_u32(qeps + ql)));
            const float num = __fsub_rd(lds_volatile_f32(smem_u32(sbound + ql)), eps[i]);
            const bool pos = num >= 0.0f;
            thrI[i] = __float2int_rd(__fmul_rd(__fmul_rd(num, pos ? rt.x : rt.y), pos ? qp.y : qp.z));
        }
        const unsigned long long c_wait = PROF ? clock64() : 0;
        wgmma_wait<0>();
        if (a.kblocks > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[prev]));
        unsigned long long c_epi = 0;
        if (PROF) {
            c_epi = clock64();
            p_turn += c_main - c_turn;
            p_full += c_full;
            p_mma += (c_thr - c_main - c_full) + (c_epi - c_wait);
            p_thr += c_wait - c_thr;
        }
        // class maxima and hit test of all four queries, with no branch between the queries so that their chains interleave
        const bool full_half = row0 + TS8_HALF <= a.n_rows;   // only the corpus' last tile can be partial
        const uint64_t left = a.n_rows > row0 ? a.n_rows - row0 : 0;
        int cm[4][NL];
        bool hit[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int l = 0; l < NL; ++l) cm[i][l] = INT_MIN;
        if (full_half) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t *v_i = acc + 64 * (i >> 1) + 2 * (i & 1);   // value (j, b) at v_i[4j + b]
                int zmax = INT_MIN;   // HAS_DEG: 0 if some accumulator of the half is exactly zero
#pragma unroll
                for (int j = 0; j < 16; ++j) {
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        int v = (int)v_i[4 * j + b];
                        if (HAS_DEG) {
                            zmax = v == 0 ? 0 : zmax;
                            v = v == 0 ? INT_MIN : v;
                        }
                        const int l = (j & (NG / 8 - 1)) * 2 + b;
                        cm[i][l] = max(cm[i][l], v);
                    }
                }
                int cmax = zmax;
#pragma unroll
                for (int l = 0; l < NL; ++l) cmax = max(cmax, cm[i][l]);
                hit[i] = cmax >= thrI[i];
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t *v_i = acc + 64 * (i >> 1) + 2 * (i & 1);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        const uint32_t col = 8 * j + 2 * (me & 3) + b;
                        const int v = (int)v_i[4 * j + b];
                        const int l = (j & (NG / 8 - 1)) * 2 + b;
                        if ((uint64_t)col < left && !(HAS_DEG && v == 0)) cm[i][l] = max(cm[i][l], v);
                    }
                }
                hit[i] = true;
            }
        }
        // |dp| < 2^31 (127^2 * D, D <= rerank_f32_max_dim()): INT_MIN only marks an empty class.
        // The lower bound fl_down(fl_down(cm * s) - eps) (s = slo for cm >= 0, shi >= slo >= 0 otherwise) does not
        // decrease with cm, so no class can grow unless the largest class maximum's bound exceeds gmin: one bound per
        // query and tile instead of NL, and the per-class fold only on the rare tiles that can raise one.
        bool grow[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t ql = qrow + 64 * (i >> 1) + 8 * (i & 1);
            hit[i] = hit[i] && mt * TS_BLOCK_M + ql < a.n_queries;
            int cmx = cm[i][0];
#pragma unroll
            for (int l = 1; l < NL; ++l) cmx = max(cmx, cm[i][l]);
            const float lbx = __fsub_rd(__fmul_rd(__int2float_rd(cmx), cmx >= 0 ? slo[i] : shi[i]), eps[i]);
            grow[i] = cmx != INT_MIN && lbx > gmin[i];
        }
        unsigned long long c_fold = 0;
        if (PROF) {
            c_fold = clock64();
            p_cmax += c_fold - c_epi;
        }
        if (__any_sync(0xffffffffu, grow[0] || grow[1] || grow[2] || grow[3])) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (!grow[i]) continue;
                const uint32_t ql = qrow + 64 * (i >> 1) + 8 * (i & 1);
                float mn = INFINITY;
#pragma unroll
                for (int l = 0; l < NL; ++l) {
                    const float lb = __fsub_rd(__fmul_rd(__int2float_rd(cm[i][l]), cm[i][l] >= 0 ? slo[i] : shi[i]), eps[i]);
                    if (cm[i][l] != INT_MIN && lb > gm[i][l]) {
                        gm[i][l] = lb;
                        red_shared_max_s32(smem_u32(cls + (8 * (l >> 1) + 2 * (me & 3) + (l & 1)) * TS_BLOCK_M + ql), f2ord(lb));
                    }
                    mn = fminf(mn, gm[i][l]);
                }
                gmin[i] = mn;
            }
        }
        unsigned long long c_emit = 0;
        if (PROF) {
            c_emit = clock64();
            p_fold += c_emit - c_fold;
        }
        if (a.emit && __any_sync(0xffffffffu, hit[0] || hit[1] || hit[2] || hit[3])) {
            const uint32_t lim = left < TS8_HALF ? (uint32_t)left : TS8_HALF;   // columns of the half that hold rows
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (!hit[i]) continue;
                const uint32_t qi = mt * TS_BLOCK_M + qrow + 64 * (i >> 1) + 8 * (i & 1);
                const uint32_t *v_i = acc + 64 * (i >> 1) + 2 * (i & 1);
                uint32_t *stage = reinterpret_cast<uint32_t *>(lstage + (size_t)(me * 4 + i) * TS8_SLOT_BYTES);
                // the passing values as a mask (bit 2j + b: column 8j + 2(me & 3) + b) without a branch per value, then
                // one emission per set bit in column order: a warp with a hit delays its warpgroup's next turn
                uint32_t pass = 0;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        const uint32_t col = 8 * j + 2 * (me & 3) + b;
                        if (col < lim && (int)v_i[4 * j + b] >= thrI[i]) pass |= 1u << (2 * j + b);
                    }
                }
                while (pass) {
                    const uint32_t x = __ffs(pass) - 1;
                    pass &= pass - 1;
                    epi_emit<TS8_LSTAGE>(a.cand, a.cand_cnt, a.cand_cap, qi, stage,
                                         a.id_base + (uint32_t)(row0 + 8 * (x >> 1) + 2 * (me & 3) + (x & 1)));
                }
            }
        }
        if (PROF) p_emit += clock64() - c_emit;
    }
    if (PROF && (ct & 127) == 0) {
        atomicAdd(a.prof + TS_PROF_MATH_WAIT, p_turn);
        atomicAdd(a.prof + TS_PROF_FULL_WAIT, p_full);
        atomicAdd(a.prof + TS_PROF_MMA, p_mma);
        atomicAdd(a.prof + TS_PROF_EPILOGUE, p_thr + p_cmax + p_fold + p_emit);
        atomicAdd(a.prof + TS_PROF_EPI_THR, p_thr);
        atomicAdd(a.prof + TS_PROF_EPI_CMAX, p_cmax);
        atomicAdd(a.prof + TS_PROF_EPI_FOLD, p_fold);
        atomicAdd(a.prof + TS_PROF_EPI_EMIT, p_emit);
        atomicAdd(a.prof + TS_PROF_TILES, (unsigned long long)T);
        atomicAdd(a.prof + TS_PROF_CONSUMER, clock64() - p_c);
    }
    // final publish + flush of the staged candidates
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t ql = 64 * (i >> 1) + 16 * wl + ((uint32_t)lane >> 2) + 8 * (i & 1), qi = mt * TS_BLOCK_M + ql;
        if (qi >= a.n_queries) continue;
#pragma unroll
        for (int l = 0; l < NL; ++l)
            atomicMax(a.ggm + (size_t)mt * NG * TS_BLOCK_M + ql + (size_t)(8 * (l >> 1) + 2 * qd + (l & 1)) * TS_BLOCK_M, f2ord(gm[i][l]));
        const uint32_t *stage = reinterpret_cast<const uint32_t *>(lstage + (size_t)(ct * 4 + i) * TS8_SLOT_BYTES);
        const uint32_t c = stage[0];
        if (a.emit && c) {
            const uint32_t pos = atomicAdd(a.cand_cnt + qi, c);
            for (uint32_t x = 0; x < c; ++x)
                if (pos + x < a.cand_cap) a.cand[(size_t)qi * a.cand_cap + pos + x] = stage[1 + x];
        }
    }
    if ((ct & 127) == 0) atomicAdd(ctl + 1, 1u);   // the bound warp stops once both warpgroups have published
}

// ------------------------------------------------------------------ fp16 normalised copies
// x_hat = x / |x| (IEEE), rounded to fp16.  Rows whose norm is outside [1e-15, 1e15] (zero, underflowed, overflowed,
// inf/NaN) are DEGENERATE: the error bound of the prefilter does not cover them, their shadow row is all zero.
// Deleted rows get an all-zero shadow row as well: like a degenerate row they then stay out of the class maxima (HAS_DEG),
// and the re-rank drops them if they are emitted.
__host__ __device__ inline bool norm_is_proper(float m) { return m >= 1.0e-15f && m <= 1.0e15f; }

// rows [first, first + n); raw / mags / out point at row `first`, `deleted` (may be null) is indexed by absolute row
__global__ void normalize_f16_kernel(const float *__restrict__ raw, uint32_t pitch_elems, const float *__restrict__ mags,
                                     uint64_t first, uint64_t n, uint32_t dim, __half *__restrict__ out, uint32_t out_pitch,
                                     const uint32_t *__restrict__ deleted) {
    const uint32_t groups = (dim + 7) / 8;
    uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= n * groups) return;
    uint64_t row = gid / groups;
    uint32_t c0 = (uint32_t)(gid % groups) * 8;
    const float m = mags[row];
    const bool ok = norm_is_proper(m) && !bit_is_set(deleted, first + row);
    for (uint32_t e = 0; e < 8 && c0 + e < dim; ++e) {
        float v = raw[row * pitch_elems + c0 + e];
        out[row * out_pitch + c0 + e] = __float2half_rn(ok ? __fdiv_rn(v, m) : 0.0f);
    }
}

cdb_status normalize_f16_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t first, uint64_t n,
                                uint32_t dim, void *d_out, uint32_t out_pitch_halfs, const uint32_t *d_deleted, cudaStream_t s) {
    if (!n) return CDB_OK;
    uint64_t total = n * ((dim + 7) / 8);
    normalize_f16_kernel<<<(uint32_t)((total + 255) / 256), 256, 0, s>>>(d_raw, pitch_elems, d_mags, first, n, dim,
                                                                          reinterpret_cast<__half *>(d_out), out_pitch_halfs, d_deleted);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// ------------------------------------------------------------------ s8 shadow (KIND 2, DESIGN.md section 5c)
__device__ __forceinline__ float warp_max_f(float v) {
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// code of one normalised entry v under scale sc (sc = 0: every v of the row set is 0)
__device__ __forceinline__ int s8_code(float v, float sc) {
    return sc > 0.0f ? max(-127, min(127, __float2int_rn(__fdiv_rn(v, sc)))) : 0;
}
// upper bound of sqrt(e2), e2 a sum of at most 2^17 f64 squares (relative rounding error < 2^-35, covered by 2^-30)
__device__ __forceinline__ float residual_norm_up(double e2) {
    return __double2float_ru(__dsqrt_ru(__dmul_ru(e2, 1.0 + 0x1p-30)));
}

// One CTA (8 warps, a warp per row) per corpus tile t = tile0 + blockIdx.x, rows [256t, min(256t + 256, row_end)):
// x_hat = x / |x| exactly as normalize_f16_kernel computes it, s_T = max |x_hat_i| / 127 over the tile's proper rows,
// codes rint(x_hat / s_T), E_T >= max over proper rows of |x_hat - s_T * codes| (f64, rounded up).  Degenerate and
// deleted rows get zero codes and no say in s_T or E_T.  tiles (may be null): the CTA's tile is tiles[blockIdx.x].
// tile_rcp[t] = {1/s_T rounded down, 1/s_T rounded up}: the s8 scan's threshold multiplies by them instead of dividing.
__global__ void __launch_bounds__(256) quantize_s8_tiles_kernel(const float *__restrict__ raw, uint32_t pitch_elems,
                                                                const float *__restrict__ mags, uint32_t tile0, uint64_t row_end,
                                                                uint32_t dim, int8_t *__restrict__ xs8, uint32_t pitch8,
                                                                float2 *__restrict__ tile_se, float2 *__restrict__ tile_rcp,
                                                                const uint32_t *__restrict__ tiles, const uint32_t *__restrict__ deleted) {
    __shared__ float s_max[8];
    __shared__ double s_e2[8];
    const uint32_t t = tiles ? tiles[blockIdx.x] : tile0 + blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t r0 = (uint64_t)t * TS_BLOCK_N, r1 = min(r0 + TS_BLOCK_N, row_end);
    float mx = 0.0f;
    for (uint64_t r = r0 + warp; r < r1; r += 8) {
        const float m = mags[r];
        if (!norm_is_proper(m) || bit_is_set(deleted, r)) continue;
        for (uint32_t c = lane; c < dim; c += 32) mx = fmaxf(mx, fabsf(__fdiv_rn(raw[r * pitch_elems + c], m)));
    }
    mx = warp_max_f(mx);
    if (lane == 0) s_max[warp] = mx;
    __syncthreads();
    mx = s_max[0];
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, s_max[w]);
    const float st = mx > 0.0f ? __fdiv_rn(mx, 127.0f) : 0.0f;
    double e2 = 0.0;
    for (uint64_t r = r0 + warp; r < r1; r += 8) {
        const float m = mags[r];
        const bool ok = norm_is_proper(m) && !bit_is_set(deleted, r);
        double rr = 0.0;
        for (uint32_t c = lane; c < dim; c += 32) {
            const float v = ok ? __fdiv_rn(raw[r * pitch_elems + c], m) : 0.0f;
            const int code = s8_code(v, st);
            xs8[r * pitch8 + c] = (int8_t)code;
            const double d = (double)v - (double)st * (double)code;
            rr += d * d;
        }
        e2 = fmax(e2, warp_sum_d(rr));
    }
    if (lane == 0) s_e2[warp] = e2;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) e2 = fmax(e2, s_e2[w]);
        tile_se[t] = make_float2(st, residual_norm_up(e2));
        tile_rcp[t] = make_float2(__frcp_rd(st), __frcp_ru(st));   // s_T = 0: +inf, see tensor_scan_s8_kernel's threshold
    }
}

// *out = max over the first ntiles tiles of E_T (the shard's E_max, read by the s8 gate)
__global__ void __launch_bounds__(1024) s8_emax_kernel(const float2 *__restrict__ tile_se, uint32_t ntiles, float *out) {
    __shared__ float s_max[32];
    float mx = 0.0f;
    for (uint32_t t = threadIdx.x; t < ntiles; t += 1024) mx = fmaxf(mx, tile_se[t].y);
    mx = warp_max_f(mx);
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = warp_max_f(s_max[threadIdx.x]);
        if (threadIdx.x == 0) *out = mx;
    }
}

cdb_status quantize_s8_device(const float *d_raw, uint32_t pitch_elems, const float *d_mags, uint64_t first, uint64_t n,
                              uint64_t row_end, uint32_t dim, void *d_xs8, uint32_t pitch8, float2 *d_tile_se, float2 *d_tile_rcp,
                              float *d_emax, const uint32_t *d_deleted, cudaStream_t s) {
    if (!n) return CDB_OK;
    const uint32_t t0 = (uint32_t)(first / TS_BLOCK_N), t1 = (uint32_t)((first + n + TS_BLOCK_N - 1) / TS_BLOCK_N);
    quantize_s8_tiles_kernel<<<t1 - t0, 256, 0, s>>>(d_raw, pitch_elems, d_mags, t0, row_end, dim,
                                                     reinterpret_cast<int8_t *>(d_xs8), pitch8, d_tile_se, d_tile_rcp, nullptr,
                                                     d_deleted);
    CDB_LAUNCH_CHECK();
    s8_emax_kernel<<<1, 1024, 0, s>>>(d_tile_se, (uint32_t)((row_end + TS_BLOCK_N - 1) / TS_BLOCK_N), d_emax);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// one CTA per listed row: the row's bytes := 0
__global__ void zero_rows_kernel(const uint32_t *__restrict__ rows, uint8_t *base, uint32_t pitch_bytes) {
    uint8_t *p = base + (size_t)rows[blockIdx.x] * pitch_bytes;
    for (uint32_t c = threadIdx.x; c < pitch_bytes; c += blockDim.x) p[c] = 0;
}

cdb_status shadow_drop_rows_device(const uint32_t *d_rows, uint32_t n_rows, const uint32_t *d_tiles, uint32_t n_tiles, void *d_xh,
                                   uint32_t xh_pitch_halfs, const float *d_raw, uint32_t pitch_elems, const float *d_mags,
                                   uint64_t row_end, uint32_t dim, void *d_xs8, uint32_t pitch8, float2 *d_tile_se, float2 *d_tile_rcp,
                                   float *d_emax, const uint32_t *d_deleted, cudaStream_t s) {
    if (n_rows) {
        zero_rows_kernel<<<n_rows, 128, 0, s>>>(d_rows, reinterpret_cast<uint8_t *>(d_xh), xh_pitch_halfs * 2);
        CDB_LAUNCH_CHECK();
    }
    if (d_xs8 && n_tiles) {
        quantize_s8_tiles_kernel<<<n_tiles, 256, 0, s>>>(d_raw, pitch_elems, d_mags, 0, row_end, dim, reinterpret_cast<int8_t *>(d_xs8),
                                                         pitch8, d_tile_se, d_tile_rcp, d_tiles, d_deleted);
        CDB_LAUNCH_CHECK();
        s8_emax_kernel<<<1, 1024, 0, s>>>(d_tile_se, (uint32_t)((row_end + TS_BLOCK_N - 1) / TS_BLOCK_N), d_emax);
        CDB_LAUNCH_CHECK();
    }
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
//   qh      fp16 copy of q / |q| (zero row for a degenerate norm and for the padding rows up to mtiles*128), or with q_se
//           (s8 form, KIND 2) s8 codes rint(q_hat / s_q) with s_q = max |q_hat_i| / 127 (qh_pitch then counts bytes) and
//           q_se = {s_q, e_q >= |q_hat - s_q * codes|}, q_rcp = {1/s_q rounded down, rounded up}
//   ggm     class maxima of the query := -inf;  cand_cnt := number of pre-seeded odd rows (+ their ids);  err := 0
//   progress counters of the seeding and of the main pass := 0
// One CTA of 128 threads per query slot (mtiles*128 slots).
__global__ void __launch_bounds__(128) prep_queries_kernel(const float *__restrict__ q, uint32_t nq, uint32_t dim, float *__restrict__ q_raw,
                                                           uint32_t raw_pitch_elems, float *__restrict__ q_mags, __half *__restrict__ qh,
                                                           uint32_t qh_pitch, int *__restrict__ ggm, const uint32_t *__restrict__ deg,
                                                           uint32_t has_deg, uint32_t id_base, uint32_t *__restrict__ cand,
                                                           uint32_t cand_cap, uint32_t *__restrict__ cand_cnt, uint32_t *__restrict__ err32,
                                                           uint8_t *__restrict__ err8, uint32_t *__restrict__ progress,
                                                           float2 *__restrict__ q_se, float2 *__restrict__ q_rcp) {
    extern __shared__ float sq[];     // [dim] squares, then (s8 form) q_hat
    __shared__ float s_mag;
    __shared__ float s_max[4];
    __shared__ double s_e2[4];
    const uint32_t slot = blockIdx.x, tid = threadIdx.x;
    if (slot == 0) for (uint32_t i = tid; i < 2048; i += 128) progress[i] = 0u;
    // class maxima: layout [tile][class][128]
    if (tid < (uint32_t)TS_GROUPS) ggm[((size_t)(slot >> 7) * TS_GROUPS + tid) * TS_BLOCK_M + (slot & 127u)] = (int)0x807FFFFF;   // f2ord(-inf)
    __half *hrow = qh + (size_t)slot * qh_pitch;
    int8_t *crow = reinterpret_cast<int8_t *>(qh) + (size_t)slot * qh_pitch;
    if (slot >= nq) {
        if (q_se) for (uint32_t c = tid; c < qh_pitch; c += 128) crow[c] = 0;
        else for (uint32_t c = tid; c < qh_pitch; c += 128) hrow[c] = __float2half_rn(0.0f);
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
    if (!q_se) {
        for (uint32_t c = tid; c < qh_pitch; c += 128)
            hrow[c] = __float2half_rn((ok && c < dim) ? __fdiv_rn(src[c], m) : 0.0f);
        return;
    }
    const uint32_t warp = tid >> 5, lane = tid & 31;
    float mx = 0.0f;
    for (uint32_t c = tid; c < dim; c += 128) {
        const float v = ok ? __fdiv_rn(src[c], m) : 0.0f;
        sq[c] = v;
        mx = fmaxf(mx, fabsf(v));
    }
    mx = warp_max_f(mx);
    if (lane == 0) s_max[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(s_max[0], s_max[1]), fmaxf(s_max[2], s_max[3]));
    const float sc = mx > 0.0f ? __fdiv_rn(mx, 127.0f) : 0.0f;
    double e2 = 0.0;
    for (uint32_t c = tid; c < qh_pitch; c += 128) {
        int code = 0;
        if (c < dim) {
            const float v = sq[c];
            code = s8_code(v, sc);
            const double d = (double)v - (double)sc * (double)code;
            e2 += d * d;
        }
        crow[c] = (int8_t)code;
    }
    e2 = warp_sum_d(e2);
    if (lane == 0) s_e2[warp] = e2;
    __syncthreads();
    if (tid == 0) {
        q_se[slot] = make_float2(sc, residual_norm_up((s_e2[0] + s_e2[1]) + (s_e2[2] + s_e2[3])));
        q_rcp[slot] = make_float2(__frcp_rd(sc), __frcp_ru(sc));
    }
}

cdb_status prep_queries_device(const float *d_q, uint32_t nq, uint32_t dim, float *d_q_raw, uint32_t raw_pitch_elems, float *d_q_mags,
                               void *d_qh, uint32_t qh_pitch_halfs, int *d_ggm, const uint32_t *d_deg, bool has_deg, uint32_t id_base,
                               uint32_t *d_cand, uint32_t cand_cap, uint32_t *d_cand_cnt, uint32_t *d_err32, uint8_t *d_err8,
                               uint32_t *d_progress, float2 *d_q_se, float2 *d_q_rcp, cudaStream_t s) {
    const uint32_t mtiles = (nq + TS_BLOCK_M - 1) / TS_BLOCK_M;
    // dim*4 bytes of squares: above 12287 dims that exceeds the 48 KB a launch gets without the opt-in
    CDB_ALLOW_SMEM(prep_queries_kernel, (size_t)dim * 4);
    prep_queries_kernel<<<mtiles * TS_BLOCK_M, 128, (size_t)dim * 4, s>>>(d_q, nq, dim, d_q_raw, raw_pitch_elems, d_q_mags,
                                                                          reinterpret_cast<__half *>(d_qh), qh_pitch_halfs, d_ggm, d_deg,
                                                                          has_deg ? 1u : 0u, id_base, d_cand, cand_cap, d_cand_cnt, d_err32,
                                                                          d_err8, d_progress, d_q_se, d_q_rcp);
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

// cdb_debug_scan_profile: launches use the instrumented instantiation while g_scan_prof_on is set
static std::atomic<bool> g_scan_prof_on{false};
static unsigned long long *g_scan_prof = nullptr;   // [TS_PROF_SLOTS] on the device that enabled profiling

template <int NG, bool HAS_DEG, int KIND>
static cdb_status launch_tensor_scan_gd(const CUtensorMap &mq, const CUtensorMap &mx, const TensorScanArgs &a, uint32_t grid,
                                        cudaStream_t s) {
    // s8 form: tensor_scan_s8_kernel for k <= 12.  At NG = 32 / 64 its 4 x NG/4 class maxima do not fit next to the 128
    // accumulators in the consumers' 232 registers (ptxas spills 24 / 536 bytes), so larger k keep the streamed kernel.
    if constexpr (KIND == 2 && NG == 16) {
        if (a.stages) {
            auto kern = tensor_scan_s8_kernel<NG, HAS_DEG, false>;
            if (a.prof) {
                if constexpr (NG == 16 && !HAS_DEG) kern = tensor_scan_s8_kernel<NG, HAS_DEG, true>;
                else { set_error("tensor scan profile: only for k <= 12 on shards without degenerate or deleted rows"); return CDB_INVALID_PARAMS; }
            }
            const size_t smem = TS8_SMEM_FIXED + (size_t)(a.kblocks + a.stages) * TS8_KB_BYTES;
            CDB_ALLOW_SMEM(kern, smem);
            kern<<<grid, TS_THREADS, smem, s>>>(mq, mx, a);
            CDB_LAUNCH_CHECK();
            return CDB_OK;
        }
    }
    auto kern = tensor_scan_kernel<TS_STAGES, NG, HAS_DEG, KIND, false>;
    if (a.prof) {   // the instrumented instantiation exists for the headline's k <= 12 without degenerate rows
        if constexpr (NG == 16 && !HAS_DEG) kern = tensor_scan_kernel<TS_STAGES, NG, HAS_DEG, KIND, true>;
        else { set_error("tensor scan profile: only for k <= 12 on shards without degenerate or deleted rows"); return CDB_INVALID_PARAMS; }
    }
    const size_t smem = tensor_scan_smem(TS_STAGES);
    CDB_ALLOW_SMEM(kern, smem);
    kern<<<grid, TS_THREADS, smem, s>>>(mq, mx, a);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

template <int NG, int KIND>
static cdb_status launch_tensor_scan_g(const CUtensorMap &mq, const CUtensorMap &mx, const TensorScanArgs &a, uint32_t grid, cudaStream_t s) {
    if constexpr (KIND == 1) return launch_tensor_scan_gd<NG, false, KIND>(mq, mx, a, grid, s);   // exact scores: no degenerate-row variant
    else return a.has_deg ? launch_tensor_scan_gd<NG, true, KIND>(mq, mx, a, grid, s)
                     : launch_tensor_scan_gd<NG, false, KIND>(mq, mx, a, grid, s);
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
    if (g_scan_prof_on.load()) a.prof = g_scan_prof;
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

// ------------------------------------------------------------------ s8 form: refilter against the final bound
// tensor_scan_s8_kernel tests every value against the bound its CTA knew at the time, and that bound only rises during the
// scan: rows of the early tiles pass against a bound far below the final one.  The test stays sound for any rigorous lower
// bound of the k-th best exact score, so it is applied once more, after the scan, against the final one (the k-th largest
// of the query's final class maxima): the value v = q_codes . x_codes (exact in s32, as the MMA computes it) and the
// threshold thrI(q, T) with the epilogue's arithmetic, rounding for rounding.  The survivors (every row of the exact
// top-k among them) are compacted to the front of the list and counted in out_cnt; the re-rank gathers their f32 rows
// only: a candidate costs 768 bytes of s8 row here instead of 3 KB of f32 row there (D = 768).  Shards without degenerate
// or deleted rows only (no pre-seeded rows, no zero shadow rows), and only the queries whose list did not overflow.
constexpr int TS8_RF_THREADS = 256;

__global__ void __launch_bounds__(TS8_RF_THREADS) s8_refilter_kernel(
    const int8_t *__restrict__ xs8, const int8_t *__restrict__ qs8, uint32_t pitch8, uint32_t dim, uint32_t k,
    const int *__restrict__ ggm, const float2 *__restrict__ tile_se, const float2 *__restrict__ tile_rcp,
    const float2 *__restrict__ q_se, const float2 *__restrict__ q_rcp, float dn1, float dref, uint32_t id_base,
    uint32_t *__restrict__ cand, const uint32_t *__restrict__ cand_cnt, uint32_t cap, uint32_t *__restrict__ out_cnt) {
    __shared__ float s_bound;
    __shared__ uint32_t s_kept;
    const uint32_t qi = blockIdx.x;
    const uint32_t cnt = cand_cnt[qi];
    if (cnt > cap) {   // the exact scan re-does this query; its list is left as it is
        if (threadIdx.x == 0) out_cnt[qi] = cap;
        return;
    }
    if (threadIdx.x == 0) {
        // the bound warp's selection (s8_bound_round) over the final class maxima
        const int *gq = ggm + (size_t)(qi / TS_BLOCK_M) * TS8_NG * TS_BLOCK_M + qi % TS_BLOCK_M;
        int v[TS8_NG];
        for (int c = 0; c < TS8_NG; ++c) v[c] = gq[c * TS_BLOCK_M];
        int b = INT_MIN;
        for (int i = 0; i < TS8_NG; ++i) {
            uint32_t n = 0;
            for (int c = 0; c < TS8_NG; ++c) n += v[c] >= v[i];
            b = n >= k ? max(b, v[i]) : b;
        }
        s_bound = ord2f(b);
        s_kept = 0;
    }
    __syncthreads();
    const float bound = s_bound;
    const float2 qse = q_se[qi], qrc = q_rcp[qi];
    const float qw = __fadd_ru(dn1, qse.y), qeps = __fmaf_ru(qse.y, dn1, dref);   // qpar.w and qeps of the scan
    const int8_t *qrow = qs8 + (size_t)qi * pitch8;
    // an 8-lane group per candidate, 16-byte loads (rows are 16-byte pitched): a round keeps 32 rows in flight per CTA
    const uint32_t grp = threadIdx.x >> 3, j = threadIdx.x & 7, vecs = dim / 16;
    for (uint32_t base = 0; base < cnt; base += TS8_RF_THREADS / 8) {
        const uint32_t ci = base + grp;
        const uint32_t id = ci < cnt ? cand[(size_t)qi * cap + ci] : CDB_INVALID_ID;
        __syncthreads();   // every id of this round is read before any survivor is written back
        const uint64_t row = id != CDB_INVALID_ID ? (uint64_t)(id - id_base) : 0;
        const int8_t *xrow = xs8 + row * pitch8;
        int dp = 0;
        if (id != CDB_INVALID_ID) {
            for (uint32_t v = j; v < vecs; v += 8) {
                const int4 x4 = reinterpret_cast<const int4 *>(xrow)[v], q4 = reinterpret_cast<const int4 *>(qrow)[v];
                dp = __dp4a(x4.x, q4.x, dp);
                dp = __dp4a(x4.y, q4.y, dp);
                dp = __dp4a(x4.z, q4.z, dp);
                dp = __dp4a(x4.w, q4.w, dp);
            }
            if (j == 0)
                for (uint32_t c = vecs * 16; c < dim; ++c) dp += (int)xrow[c] * (int)qrow[c];
        }
        // integer sums: exact in any order, the value the MMA accumulated
        dp += __shfl_xor_sync(0xFFFFFFFFu, dp, 1);
        dp += __shfl_xor_sync(0xFFFFFFFFu, dp, 2);
        dp += __shfl_xor_sync(0xFFFFFFFFu, dp, 4);
        if (j == 0 && id != CDB_INVALID_ID) {
            const uint64_t nt = row / TS_BLOCK_N;
            const float2 se = tile_se[nt], rt = tile_rcp[nt];
            const float eps = __fmaf_ru(qw, se.y, qeps);
            const float num = __fsub_rd(bound, eps);
            const bool pos = num >= 0.0f;
            const int thr = __float2int_rd(__fmul_rd(__fmul_rd(num, pos ? rt.x : rt.y), pos ? qrc.x : qrc.y));
            if (dp >= thr) cand[(size_t)qi * cap + atomicAdd(&s_kept, 1u)] = id;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) out_cnt[qi] = s_kept;
}


// smallest float >= x
static float f32_up(double x) {
    float f = (float)x;
    return (double)f < x ? std::nextafter(f, INFINITY) : f;
}

// s8 form (KIND 2, DESIGN.md section 5c): d_xs8 s8 shadow [n_rows][pitch8], d_qs8 query codes padded with zero rows to a
// multiple of 128, d_tile_se / d_q_se their {scale, residual bound}, d_tile_rcp / d_q_rcp the scales' reciprocals.  Same candidates / class maxima contract as
// tensor_scan_device; prep_queries_device (s8 mode) has reset them.
cdb_status tensor_scan_s8_device(const void *d_xs8, const void *d_qs8, uint32_t pitch8, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, const float2 *d_tile_se, const float2 *d_tile_rcp, const float2 *d_q_se,
                                 const float2 *d_q_rcp, uint32_t id_base, int *d_ggm,
                                 uint32_t *d_cand, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_progress, bool has_deg,
                                 int sm_count, cudaStream_t s, uint32_t *d_kept_cnt, bool *refiltered) {
    TensorScanArgs a{};
    a.has_deg = has_deg ? 1u : 0u;
    a.window = 3;
    a.refresh_mask = 15;
    if (const char *e = getenv("CDB_TS_WINDOW")) a.window = (uint32_t)atoi(e);
    if (const char *e = getenv("CDB_TS_REFRESH")) a.refresh_mask = (uint32_t)atoi(e);
    a.n_rows = n_rows;
    a.n_queries = nq;
    a.k = k;
    a.kblocks = (dim + 2 * TS_BLOCK_K - 1) / (2 * TS_BLOCK_K);   // 128 s8 elements per 128-byte row
    a.mtiles = (nq + TS_BLOCK_M - 1) / TS_BLOCK_M;
    a.ntiles = (uint32_t)((n_rows + TS_BLOCK_N - 1) / TS_BLOCK_N);
    a.id_base = id_base;
    a.ggm = d_ggm;
    a.cand = d_cand;
    a.cand_cnt = d_cand_cnt;
    a.cand_cap = cand_cap;
    a.tile_se = d_tile_se;
    a.tile_rcp = d_tile_rcp;
    a.q_se = d_q_se;
    a.q_rcp = d_q_rcp;
    // u = 2^-24.  |x_hat|, |q_hat| <= 1 + (D/2 + 2) u + O(D^2 u^2) (sequential f32 norm, one division per entry);
    // |cos_ref - q_hat . x_hat| <= (D + 4) u + O(D^2 u^2) (FMA dot product, norm product, division).  Both are taken
    // twice over, which covers the second-order terms for every D <= rerank_f32_max_dim().
    a.dn1 = f32_up(1.0 + ((double)dim + 8.0) * 0x1p-24);
    a.dref = f32_up((2.0 * dim + 16.0) * 0x1p-24);
    a.rel = 1.0f;
    if (!tensor_scan_stages(k)) { set_error("s8 tensor scan: k too large (class-maximum bound needs k <= 64)"); return CDB_INVALID_PARAMS; }
    // tensor_scan_s8_kernel for k <= 12 (NG = 16, see launch_tensor_scan_gd) while the resident query tile leaves room for
    // TS8_MIN_STAGES corpus stages (D <= 1024), else the streamed tensor_scan_kernel.  The two take differently shaped
    // corpus boxes (128 / 256 rows), so a.stages != 0 must mean exactly "the s8 kernel runs".
    const size_t room = 227 * 1024 - TS8_SMEM_FIXED;
    const uint32_t fit = (uint32_t)(room / TS8_KB_BYTES) > a.kblocks ? (uint32_t)(room / TS8_KB_BYTES) - a.kblocks : 0;
    a.stages = k <= 12 && fit >= TS8_MIN_STAGES ? std::min(fit, TS8_MAX_STAGES) : 0;
    CUtensorMap mq, mx;
    cdb_status rc;
    if ((rc = make_tensor_map_2d(&mq, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, d_qs8, (uint64_t)a.mtiles * TS_BLOCK_M, dim, pitch8, TS_BLOCK_M))) return rc;
    if ((rc = make_tensor_map_2d(&mx, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, d_xs8, n_rows, dim, pitch8, a.stages ? TS8_HALF : TS_BLOCK_N))) return rc;
    if ((rc = run_tensor_scan<2>(mq, mx, a, n_rows, d_progress, sm_count, s))) return rc;
    *refiltered = d_kept_cnt && a.stages && !has_deg;
    if (!*refiltered) return CDB_OK;
    s8_refilter_kernel<<<nq, TS8_RF_THREADS, 0, s>>>(static_cast<const int8_t *>(d_xs8), static_cast<const int8_t *>(d_qs8), pitch8,
                                                     dim, k, d_ggm, d_tile_se, d_tile_rcp, d_q_se, d_q_rcp, a.dn1, a.dref, id_base,
                                                     d_cand, d_cand_cnt, cand_cap, d_kept_cnt);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

// Integer form (tensor_scan_u8.cu): d_x u8 operand rows [n_rows][pitch] (u8 codes or unpacked digits), d_q the query operand
// rows padded with zero rows to a multiple of 128.  Emits exact selection keys into d_cand64; the caller sorts them.
cdb_status tensor_scan_i8_device(const uint8_t *d_x, const uint8_t *d_q, uint32_t pitch, uint64_t n_rows, uint32_t nq, uint32_t dim,
                                 uint32_t k, int metric, const float *d_mags, const float *d_qmags, uint32_t id_base, int *d_ggm,
                                 uint64_t *d_cand64, uint32_t *d_cand_cnt, uint32_t cand_cap, uint32_t *d_err32, uint32_t *d_progress,
                                 const uint32_t *d_deleted, int sm_count, cudaStream_t s) {
    TensorScanArgs a{};
    a.deleted = d_deleted;
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

// Measurement switch of the prefilter scan (tools/bench_prefilter_resident.py; not part of the public header).  enable != 0
// runs the clock64-instrumented instantiation (k <= 12, no degenerate or deleted rows) from now on, 0 the default one;
// results are the same either way.  out (may be null, TS_PROF_SLOTS entries, see the TS_PROF_* enum) receives the sums
// accumulated since the previous call, which zeroes them.  Process-wide; synchronizes the current device, whose searches
// the profile then covers.
extern "C" cdb_status cdb_debug_scan_profile(int32_t enable, uint64_t *out) {
    using namespace cdb;
    CDB_CUDA_TRY(cudaDeviceSynchronize());
    if (out) {
        for (int i = 0; i < TS_PROF_SLOTS; ++i) out[i] = 0;
        if (g_scan_prof) CDB_CUDA_TRY(cudaMemcpy(out, g_scan_prof, TS_PROF_SLOTS * 8, cudaMemcpyDeviceToHost));
    }
    if (enable && !g_scan_prof) CDB_CUDA_TRY(cudaMalloc(&g_scan_prof, TS_PROF_SLOTS * 8));
    if (g_scan_prof) CDB_CUDA_TRY(cudaMemset(g_scan_prof, 0, TS_PROF_SLOTS * 8));
    g_scan_prof_on.store(enable != 0);
    return CDB_OK;
}
