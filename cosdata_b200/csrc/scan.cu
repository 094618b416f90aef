// scan.cu -- exact brute-force scan with fused per-query top-k (S1, BRUTE modes).
//
// Two kernels share one top-k scheme:
//   scan_f32_kernel   raw / F32 rows, cosine.  Two threads per row: thread t owns AVX
//                     lanes 4t..4t+3 of the reference's dot_product_f32_simd
//                     (x86_64.rs:418-444) and walks the row with 128-bit loads, so every
//                     (query,row) dot is bit-identical to the reference.  R rows x QB
//                     queries are register-blocked per thread.
//   scan_generic_kernel  every other (metric, storage) arm through pair_distance():
//                     one thread per row, reference operation order.
// Grid: x = query group (QB queries), y = row split.  Splits interleave 256-row
// passes, so all resident CTAs sweep the corpus front to back together and the
// query groups of one split share rows through L2.
//
// Top-k: per CTA and query a shared-memory candidate buffer guarded by a threshold
// (the k-th best key seen at the last compaction).  Scores below the threshold --
// almost all of them after warm-up -- cost one compare.  A warp compacts a buffer by
// rank selection when it could overflow.  Keys are (order_key<<32 | ~id): unique, so
// the result is the exact top-k under (score desc, id asc) whatever the arrival order.
#include "kernels.h"

namespace cdb {

constexpr int SCAN_THREADS = 256;
constexpr int RPP = 256;  // rows per pass per CTA

struct TopK {
    uint64_t *thr;  // [QB]
    int *cnt;       // [QB]
    int *err;       // [QB]
    uint64_t *buf;  // [QB][cap]
    uint64_t *tmp;  // [QB][k]
    uint32_t cap, k;
};

__host__ __device__ inline uint32_t topk_cap(uint32_t k) { return k + 3 * RPP; }
__host__ __device__ inline size_t topk_smem_bytes(uint32_t qb, uint32_t k) {
    return (size_t)qb * (8 + 4 + 4) + (size_t)qb * (topk_cap(k) + k) * 8 + 16;
}

__device__ inline TopK topk_carve(uint8_t *p, uint32_t qb, uint32_t k) {
    TopK t;
    t.cap = topk_cap(k);
    t.k = k;
    t.buf = reinterpret_cast<uint64_t *>(p);
    t.tmp = t.buf + (size_t)qb * t.cap;
    t.thr = t.tmp + (size_t)qb * k;
    t.cnt = reinterpret_cast<int *>(t.thr + qb);
    t.err = t.cnt + qb;
    return t;
}
__device__ inline void topk_init(const TopK &t, uint32_t qb) {
    for (uint32_t i = threadIdx.x; i < qb; i += blockDim.x) { t.thr[i] = 0; t.cnt[i] = 0; t.err[i] = 0; }
}
__device__ __forceinline__ bool row_deleted(const uint32_t *deleted, uint64_t row) {
    return deleted && ((deleted[row >> 5] >> (row & 31)) & 1u);
}
// a deleted row is never offered: the bitmap is read only for keys that pass the threshold, so the per-row cost stays one compare
__device__ inline void topk_offer(const TopK &t, int b, uint64_t key, const uint32_t *deleted, uint64_t row) {
    if (key > t.thr[b] && !row_deleted(deleted, row)) {
        int pos = atomicAdd(&t.cnt[b], 1);
        t.buf[(size_t)b * t.cap + pos] = key;
    }
}
// whole CTA: keep the best min(n,k) keys of buffer b, sorted best-first (rank selection: keys are unique).  All threads
// of the block must call it; buffers are processed one after the other with all 256 threads on each -- a single warp per
// buffer made the final compaction of a short scan (few passes per CTA, cold threshold, ~700 entries) cost more than the
// scan itself (84 us for 100k x 128 at batch 1).
__device__ inline void topk_compact_block(const TopK &t, int b) {
    const int n = t.cnt[b];
    uint64_t *B = t.buf + (size_t)b * t.cap;
    uint64_t *T = t.tmp + (size_t)b * t.k;
    for (int idx = threadIdx.x; idx < n; idx += SCAN_THREADS) {
        const uint64_t key = B[idx];
        uint32_t rank = 0;
        for (int j = 0; j < n; ++j) rank += (B[j] > key);
        if (rank < t.k) T[rank] = key;
    }
    __syncthreads();
    const int m = n < (int)t.k ? n : (int)t.k;
    for (int idx = threadIdx.x; idx < m; idx += SCAN_THREADS) B[idx] = T[idx];
    if (threadIdx.x == 0) {
        t.cnt[b] = m;
        if (n >= (int)t.k) t.thr[b] = T[t.k - 1];
    }
    __syncthreads();
}
// end of a pass: compacts when a buffer could overflow during the next pass.
// A reader may miss appends of the current pass (<= RPP), hence the slack in topk_cap().
__device__ inline void topk_end_pass(const TopK &t, uint32_t qb) {
    int pred = (threadIdx.x < qb) ? (t.cnt[threadIdx.x] > (int)(t.k + RPP)) : 0;
    if (__syncthreads_or(pred)) {
        for (uint32_t b = 0; b < qb; ++b)
            if (t.cnt[b] > (int)t.k) topk_compact_block(t, (int)b);   // block-uniform condition (shared memory, after the barrier)
    }
}
// qslot0 = first slot of this CTA's queries in the partial buffer; err goes to the real query index (qidx, may be null)
__device__ inline void topk_finish(const TopK &t, uint32_t qb, uint32_t nqv, uint32_t qslot0, uint32_t split,
                                   uint32_t nsplit, uint64_t *partial, uint32_t *err32, const uint32_t *qidx) {
    __syncthreads();
    for (uint32_t b = 0; b < qb; ++b) topk_compact_block(t, (int)b);
    for (uint32_t idx = threadIdx.x; idx < nqv * t.k; idx += blockDim.x) {
        uint32_t b = idx / t.k, j = idx % t.k;
        partial[((size_t)(qslot0 + b) * nsplit + split) * t.k + j] = (int)j < t.cnt[b] ? t.buf[(size_t)b * t.cap + j] : 0ull;
    }
    if (err32 && threadIdx.x < nqv && t.err[threadIdx.x])
        atomicOr(err32 + (qidx ? qidx[qslot0 + threadIdx.x] : qslot0 + threadIdx.x), (uint32_t)t.err[threadIdx.x]);
}

// Work assignment of one CTA (see ScanArgs).  Returns false when the CTA has nothing to do.
struct ScanWork {
    uint32_t q0, nqv, split, nsplit;
    const uint32_t *qidx;   // null: query index = slot
};
template <int QB>
__device__ __forceinline__ bool scan_work(const ScanArgs &a, ScanWork &w) {
    if (a.sel_mode) {
        const uint32_t n_sel = a.qsel[0];
        if (n_sel == 0 || n_sel > a.sel_cap) return false;
        const uint32_t groups = (n_sel + QB - 1) / QB;
        const uint32_t grp = blockIdx.x % groups;
        w.split = blockIdx.x / groups;
        w.nsplit = gridDim.x / groups;
        if (w.split >= w.nsplit) return false;
        w.q0 = grp * QB;
        w.nqv = min((uint32_t)QB, n_sel - w.q0);
        w.qidx = a.qsel + 1;
        return true;
    }
    if (a.qsel && a.qsel[0] <= a.sel_cap) return false;   // the prefilter result stands (or the selective scan handles it)
    w.q0 = blockIdx.x * QB;
    w.nqv = min((uint32_t)QB, a.nq - w.q0);
    w.split = blockIdx.y;
    w.nsplit = gridDim.y;
    w.qidx = nullptr;
    return true;
}

// ------------------------------------------------------------------ f32 exact scan
template <int QB, int R>
__global__ void __launch_bounds__(SCAN_THREADS, 2) scan_f32_kernel(ScanArgs a) {
    ScanWork w;
    if (!scan_work<QB>(a, w)) return;  // device-side decision: the prefilter succeeded, nothing to redo
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t qp = a.row_pitch / 4;  // floats per (padded) query row
    float *qs = reinterpret_cast<float *>(smem);
    float *qmag = qs + (size_t)QB * qp;
    TopK tk = topk_carve(reinterpret_cast<uint8_t *>(qmag + ((QB + 3) & ~3)), QB, a.k);

    const int tid = threadIdx.x, t = tid & 1, pi = tid >> 1;
    const uint32_t nqv = w.nqv;
    for (uint32_t i = tid; i < QB * qp; i += SCAN_THREADS) {
        uint32_t b = i / qp, c = i % qp;
        const uint32_t qi = b < nqv ? (w.qidx ? w.qidx[w.q0 + b] : w.q0 + b) : 0;
        qs[i] = (b < nqv && c < a.dim) ? reinterpret_cast<const float *>(a.q + (size_t)qi * a.row_pitch)[c] : 0.0f;
    }
    if (tid < QB) qmag[tid] = tid < (int)nqv ? a.qmags[w.qidx ? w.qidx[w.q0 + tid] : w.q0 + tid] : 0.0f;
    topk_init(tk, QB);
    __syncthreads();

    const uint32_t chunks = a.dim / 8;
    const uint64_t npass = (a.n + RPP - 1) / RPP;
    for (uint64_t pass = w.split; pass < npass; pass += w.nsplit) {
        uint64_t row[R];
        const float *xp[R];
#pragma unroll
        for (int rr = 0; rr < R; ++rr) {
            row[rr] = pass * RPP + pi + (uint64_t)(RPP / R) * rr;
            uint64_t rc = row[rr] < a.n ? row[rr] : 0;
            xp[rr] = reinterpret_cast<const float *>(a.rows + rc * a.row_pitch) + 4 * t;
        }
        float acc[R][QB][4];
#pragma unroll
        for (int rr = 0; rr < R; ++rr)
#pragma unroll
            for (int b = 0; b < QB; ++b)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[rr][b][e] = 0.0f;

        const float *qt = qs + 4 * t;
        uint32_t i = 0;
        for (; i + 2 <= chunks; i += 2) {
            float4 xv[2][R];
#pragma unroll
            for (int u = 0; u < 2; ++u)
#pragma unroll
                for (int rr = 0; rr < R; ++rr) {
                    uint4 w = ldg128_stream(xp[rr] + 8 * (i + u));
                    xv[u][rr] = make_float4(__uint_as_float(w.x), __uint_as_float(w.y), __uint_as_float(w.z), __uint_as_float(w.w));
                }
#pragma unroll
            for (int u = 0; u < 2; ++u)
#pragma unroll
                for (int b = 0; b < QB; ++b) {
                    const float4 qv = *reinterpret_cast<const float4 *>(qt + (size_t)b * qp + 8 * (i + u));
#pragma unroll
                    for (int rr = 0; rr < R; ++rr) {
                        acc[rr][b][0] = __fmaf_rn(qv.x, xv[u][rr].x, acc[rr][b][0]);
                        acc[rr][b][1] = __fmaf_rn(qv.y, xv[u][rr].y, acc[rr][b][1]);
                        acc[rr][b][2] = __fmaf_rn(qv.z, xv[u][rr].z, acc[rr][b][2]);
                        acc[rr][b][3] = __fmaf_rn(qv.w, xv[u][rr].w, acc[rr][b][3]);
                    }
                }
        }
        for (; i < chunks; ++i) {
#pragma unroll
            for (int rr = 0; rr < R; ++rr) {
                uint4 w = ldg128_stream(xp[rr] + 8 * i);
#pragma unroll
                for (int b = 0; b < QB; ++b) {
                    const float4 qv = *reinterpret_cast<const float4 *>(qt + (size_t)b * qp + 8 * i);
                    acc[rr][b][0] = __fmaf_rn(qv.x, __uint_as_float(w.x), acc[rr][b][0]);
                    acc[rr][b][1] = __fmaf_rn(qv.y, __uint_as_float(w.y), acc[rr][b][1]);
                    acc[rr][b][2] = __fmaf_rn(qv.z, __uint_as_float(w.z), acc[rr][b][2]);
                    acc[rr][b][3] = __fmaf_rn(qv.w, __uint_as_float(w.w), acc[rr][b][3]);
                }
            }
        }
        // hadd tree: thread t holds (s[4t]+s[4t+1]) + (s[4t+2]+s[4t+3]); partner adds the other half
#pragma unroll
        for (int rr = 0; rr < R; ++rr) {
            const bool valid = row[rr] < a.n;
            const float rmag = valid ? a.mags[row[rr]] : 1.0f;
            const float *xrow = xp[rr] - 4 * t;
#pragma unroll
            for (int b = 0; b < QB; ++b) {
                float h = __fadd_rn(__fadd_rn(acc[rr][b][0], acc[rr][b][1]), __fadd_rn(acc[rr][b][2], acc[rr][b][3]));
                float o = __shfl_xor_sync(0xFFFFFFFFu, h, 1);
                float tot = t == 0 ? __fadd_rn(h, o) : __fadd_rn(o, h);
                for (uint32_t c = chunks * 8; c < a.dim; ++c) tot = __fadd_rn(tot, __fmul_rn(qs[(size_t)b * qp + c], __ldg(xrow + c)));
                if (valid && (uint32_t)b < nqv && (b & 1) == t) {
                    const float denom = __fmul_rn(qmag[b], rmag);
                    if (!a.raw_mode && denom == 0.0f) {
                        if (!row_deleted(a.deleted, row[rr])) atomicOr(&tk.err[b], CDB_ERRFLAG_CALCULATION);
                    } else {
                        const float v = canon_nan(__fdiv_rn(tot, denom));
                        topk_offer(tk, b, make_key64(order_key(CDB_METRIC_COSINE, __float_as_uint(v)), a.id_base + (uint32_t)row[rr]),
                                   a.deleted, row[rr]);
                    }
                }
            }
        }
        topk_end_pass(tk, QB);
    }
    topk_finish(tk, QB, nqv, w.q0, w.split, a.sel_mode ? gridDim.x : a.nsplit, a.partial, a.err32, w.qidx);
}

// ------------------------------------------------------------------ generic scan
template <int QB>
__global__ void __launch_bounds__(SCAN_THREADS, 2) scan_generic_kernel(ScanArgs a) {
    ScanWork w;
    if (!scan_work<QB>(a, w)) return;
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t *qs = smem;  // [QB][row_pitch]
    float *qmag = reinterpret_cast<float *>(qs + (size_t)QB * a.row_pitch);
    TopK tk = topk_carve(reinterpret_cast<uint8_t *>(qmag + ((QB + 3) & ~3)), QB, a.k);
    const int tid = threadIdx.x;
    const uint32_t nqv = w.nqv;
    for (uint32_t i = tid; i < QB * (a.row_pitch / 4); i += SCAN_THREADS) {
        uint32_t b = i / (a.row_pitch / 4), c = i % (a.row_pitch / 4);
        const uint32_t qi = b < nqv ? (w.qidx ? w.qidx[w.q0 + b] : w.q0 + b) : 0;
        reinterpret_cast<uint32_t *>(qs)[i] = b < nqv ? reinterpret_cast<const uint32_t *>(a.q + (size_t)qi * a.row_pitch)[c] : 0u;
    }
    if (tid < QB) qmag[tid] = tid < (int)nqv ? a.qmags[w.qidx ? w.qidx[w.q0 + tid] : w.q0 + tid] : 0.0f;
    topk_init(tk, QB);
    __syncthreads();
    const uint32_t pp = plane_pitch(a.dim);
    const uint64_t npass = (a.n + RPP - 1) / RPP;
    for (uint64_t pass = w.split; pass < npass; pass += w.nsplit) {
        const uint64_t row = pass * RPP + tid;
        if (row < a.n) {
            const uint8_t *xr = a.rows + row * a.row_pitch;
            const float rmag = a.mags[row];
            for (uint32_t b = 0; b < nqv; ++b) {
                float v;
                int rc = pair_distance(a.metric, a.st, a.dim, qs + (size_t)b * a.row_pitch, qmag[b], pp, xr, rmag, pp, &v);
                if (rc == CDB_OK)
                    topk_offer(tk, b, make_key64(order_key(a.metric, __float_as_uint(v)), a.id_base + (uint32_t)row), a.deleted, row);
                else if (rc == CDB_CALCULATION_ERROR && !row_deleted(a.deleted, row))
                    atomicOr(&tk.err[b], CDB_ERRFLAG_CALCULATION);
            }
        }
        topk_end_pass(tk, QB);
    }
    topk_finish(tk, QB, nqv, w.q0, w.split, a.sel_mode ? gridDim.x : a.nsplit, a.partial, a.err32, w.qidx);
}

// ------------------------------------------------------------------ planning / launch
static int pick_qb(uint32_t nq, uint32_t row_pitch, uint32_t k) {
    int qb = nq >= 5 ? 8 : (nq >= 3 ? 4 : (nq == 2 ? 2 : 1));
    while (qb > 1 && (size_t)qb * row_pitch + topk_smem_bytes(qb, k) + 64 > 100 * 1024) qb >>= 1;
    return qb;
}
static size_t scan_smem(int qb, uint32_t row_pitch, uint32_t k) {
    return (size_t)qb * row_pitch + ((qb + 3) & ~3) * 4 + topk_smem_bytes(qb, k);
}

uint32_t scan_plan_nsplit(const ScanArgs &a, int sm_count) {
    const int qb = pick_qb(a.nq, a.row_pitch, a.k);
    const uint64_t ngroups = (a.nq + qb - 1) / qb;
    const uint64_t npass = (a.n + RPP - 1) / RPP;
    const uint64_t resident = 2ull * sm_count;
    uint64_t max_split = npass < 1 ? 1 : npass;
    if (max_split > 8192 / a.k) max_split = 8192 / a.k ? 8192 / a.k : 1;
    if (max_split > 1024) max_split = 1024;
    // aim for ~8 waves worth of CTAs, whole waves preferred
    uint64_t best = 1;
    double best_score = -1.0;
    for (uint64_t s = 1; s <= max_split; ++s) {
        uint64_t total = s * ngroups;
        uint64_t waves = (total + resident - 1) / resident;
        double eff = (double)total / (double)(waves * resident);
        if (waves > 8) eff *= 8.0 / (double)waves;  // do not shred the work needlessly
        if (npass / s < 4 && s > 1) eff *= 0.5;       // keep a few passes per CTA
        if (eff > best_score + 1e-9) { best_score = eff; best = s; }
    }
    return (uint32_t)best;
}

template <int QB>
static cdb_status launch_scan(const ScanArgs &a, uint32_t sel_grid, cudaStream_t s) {
    const uint32_t ngroups = (a.nq + QB - 1) / QB;
    dim3 grid(ngroups, a.nsplit);
    if (a.sel_mode) {
        if (!sel_grid) { set_error("scan: selective mode needs sel_grid"); return CDB_INVALID_PARAMS; }
        grid = dim3(sel_grid, 1);
    }
    size_t smem = scan_smem(QB, a.row_pitch, a.k);
    const bool f32path = (a.st == CDB_ST_F32 && a.metric == CDB_METRIC_COSINE);
    const void *kern = f32path ? reinterpret_cast<const void *>(scan_f32_kernel<QB, 2>)
                               : reinterpret_cast<const void *>(scan_generic_kernel<QB>);
    // the query rows and the candidate buffers live in shared memory: past the device's per-block limit no plan exists
    // (the launch would fail), so the search is refused
    int dev = 0, optin = 0;
    CDB_CUDA_TRY(cudaGetDevice(&dev));
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    cudaFuncAttributes fa;
    CDB_CUDA_TRY(cudaFuncGetAttributes(&fa, kern));
    if (smem + fa.sharedSizeBytes > (size_t)optin) {
        set_error("exact scan: dimension " + std::to_string(a.dim) + " with k " + std::to_string(a.k) + " needs " +
                  std::to_string(smem + fa.sharedSizeBytes) + " bytes of shared memory per block, the device allows " +
                  std::to_string(optin));
        return CDB_INVALID_PARAMS;
    }
    CDB_ALLOW_SMEM(kern, smem);
    if (f32path) scan_f32_kernel<QB, 2><<<grid, SCAN_THREADS, smem, s>>>(a);
    else scan_generic_kernel<QB><<<grid, SCAN_THREADS, smem, s>>>(a);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

uint32_t scan_sel_grid(int sm_count, uint32_t k) {   // the merge holds grid*k keys in shared memory
    const uint32_t lim = 16384u / (k ? k : 1u);   // padded to a power of two for the bitonic merge: <= 128 KB
    const uint32_t g = 2u * (uint32_t)sm_count;
    return g < lim ? g : (lim ? lim : 1u);
}
uint32_t scan_sel_qb(const ScanArgs &a) { return (uint32_t)pick_qb(SCAN_SEL_CAP, a.row_pitch, a.k); }

cdb_status scan_topk_device(const ScanArgs &a, cudaStream_t s) {
    if (a.k == 0 || a.k > 1024) { set_error("scan: k must be in 1..1024"); return CDB_INVALID_PARAMS; }
    if (a.nq == 0) return CDB_OK;
    // the selective scan is planned for SCAN_SEL_CAP queries whatever the batch size
    const uint32_t sel_grid = a.sel_grid;
    switch (pick_qb(a.sel_mode ? SCAN_SEL_CAP : a.nq, a.row_pitch, a.k)) {
    case 8: return launch_scan<8>(a, sel_grid, s);
    case 4: return launch_scan<4>(a, sel_grid, s);
    case 2: return launch_scan<2>(a, sel_grid, s);
    default: return launch_scan<1>(a, sel_grid, s);
    }
}

// ------------------------------------------------------------------ merge
// one CTA per query: rank-select the best k of nlists*k keys (0 = empty).
// Fallback forms (see ScanArgs): sel_mode 1 -> CTA i handles selected query qsel[1+i], whose lists are the first
// (sel_grid / groups) of a stride of sel_grid; sel_mode 0 with qsel -> runs only if n_sel > sel_cap.
__global__ void merge_partials_kernel(int metric, const uint64_t *__restrict__ partial, uint32_t nlists, uint32_t k,
                                      uint32_t *__restrict__ ids, float *__restrict__ scores, uint32_t *__restrict__ counts,
                                      const uint32_t *__restrict__ qsel, uint32_t sel_cap, int sel_mode, uint32_t sel_grid,
                                      uint32_t sel_qb, uint64_t *__restrict__ out_keys) {
    uint32_t q = blockIdx.x, stride = nlists;
    if (sel_mode) {
        const uint32_t n_sel = qsel[0];
        if (n_sel == 0 || n_sel > sel_cap || blockIdx.x >= n_sel) return;
        q = qsel[1 + blockIdx.x];
        stride = sel_grid;
        nlists = sel_grid / ((n_sel + sel_qb - 1) / sel_qb);
    } else if (qsel && qsel[0] <= sel_cap) {
        return;
    }
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem);
    __shared__ int nvalid;
    const uint32_t M = nlists * k;
    const uint64_t *src = partial + (size_t)blockIdx.x * stride * k;
    if (threadIdx.x == 0) nvalid = 0;
    for (uint32_t j = threadIdx.x; j < k; j += blockDim.x) {
        ids[(size_t)q * k + j] = CDB_INVALID_ID;
        scores[(size_t)q * k + j] = 0.0f;
        if (out_keys) out_keys[(size_t)q * k + j] = 0ull;
    }
    __syncthreads();
    int local = 0;
    for (uint32_t i = threadIdx.x; i < M; i += blockDim.x) {
        uint64_t v = src[i];
        keys[i] = v;
        local += v != 0;
    }
    if (local) atomicAdd(&nvalid, local);
    __syncthreads();
    if (M <= 768) {
        // rank selection: O(M^2 / threads)
        for (uint32_t i = threadIdx.x; i < M; i += blockDim.x) {
            const uint64_t key = keys[i];
            if (!key) continue;
            uint32_t rank = 0;
            for (uint32_t j = 0; j < M; ++j) rank += keys[j] > key;
            if (rank < k) {
                ids[(size_t)q * k + rank] = key64_id(key);
                scores[(size_t)q * k + rank] = __uint_as_float(key_to_bits(metric, (uint32_t)(key >> 32)));
                if (out_keys) out_keys[(size_t)q * k + rank] = key;
            }
        }
    } else {
        // many lists (a short scan split over every SM): bitonic sort in shared memory, O(M log^2 M / threads) -- the
        // quadratic selection took 342 us for 391 lists x 10 (batch 1 over 100k rows)
        uint32_t P = 1;
        while (P < M) P <<= 1;
        for (uint32_t i = M + threadIdx.x; i < P; i += blockDim.x) keys[i] = 0ull;
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
        const uint32_t nout = min((uint32_t)nvalid, k);
        for (uint32_t i = threadIdx.x; i < nout; i += blockDim.x) {
            const uint64_t key = keys[i];
            ids[(size_t)q * k + i] = key64_id(key);
            scores[(size_t)q * k + i] = __uint_as_float(key_to_bits(metric, (uint32_t)(key >> 32)));
            if (out_keys) out_keys[(size_t)q * k + i] = key;
        }
    }
    if (threadIdx.x == 0 && counts) counts[q] = (uint32_t)nvalid < k ? (uint32_t)nvalid : k;
}

cdb_status merge_partials_device(int metric, const uint64_t *d_partial, uint32_t nq, uint32_t nlists, uint32_t k,
                                 uint32_t *d_ids, float *d_scores, uint32_t *d_counts, cudaStream_t s, const uint32_t *qsel,
                                 uint32_t sel_cap, int sel_mode, uint32_t sel_grid, uint32_t sel_qb, uint64_t *d_out_keys) {
    if (nq == 0) return CDB_OK;
    size_t M = (size_t)(sel_mode ? sel_grid : nlists) * k, P = 1;
    while (P < M) P <<= 1;
    size_t smem = (M <= 768 ? M : P) * 8;
    if (smem > 200 * 1024) { set_error("merge: too many partial candidates"); return CDB_INVALID_PARAMS; }
    CDB_ALLOW_SMEM(merge_partials_kernel, smem);
    merge_partials_kernel<<<sel_mode ? sel_cap : nq, 256, smem, s>>>(metric, d_partial, nlists, k, d_ids, d_scores, d_counts, qsel,
                                                                      sel_cap, sel_mode, sel_grid, sel_qb, d_out_keys);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

__global__ void pack_keys_kernel(int metric, const uint32_t *ids, const float *scores, uint32_t n_shards, uint32_t nq,
                                 uint32_t k, uint64_t *keys) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t total = (uint64_t)n_shards * nq * k;
    if (i >= total) return;
    uint32_t j = (uint32_t)(i % k);
    uint32_t q = (uint32_t)((i / k) % nq);
    uint32_t sh = (uint32_t)(i / ((uint64_t)k * nq));
    uint32_t id = ids[i];
    uint64_t key = id == CDB_INVALID_ID ? 0ull : make_key64(order_key(metric, __float_as_uint(scores[i])), id);
    keys[((size_t)q * n_shards + sh) * k + j] = key;
}
cdb_status pack_keys_device(int metric, const uint32_t *d_ids, const float *d_scores, uint32_t n_shards, uint32_t nq,
                            uint32_t k, uint64_t *d_keys, cudaStream_t s) {
    uint64_t total = (uint64_t)n_shards * nq * k;
    if (!total) return CDB_OK;
    pack_keys_kernel<<<(uint32_t)((total + 255) / 256), 256, 0, s>>>(metric, d_ids, d_scores, n_shards, nq, k, d_keys);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // namespace cdb
