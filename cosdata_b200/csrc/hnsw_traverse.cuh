// hnsw_traverse.cuh -- traverse_find_nearest (src/vector_store.rs:1112-1204) for one CTA, shared by the metadata search
// kernel (hnsw_md.cu) and the index builder (hnsw_build.cu).
//
// The reference's BinaryHeap is unbounded but performs exactly `ef` pops, so an entry ranked below the number of
// pops still to come can never be popped: the queue is a sorted array of at most `ef` entries in shared memory and
// the pop order is identical to the heap's.  Keys are (order_key(score) << 32 | ~id): better score first, then
// smaller id (the oracle's tie rule where the reference's (MetricResult, pointer) order is unspecified).
#pragma once
#include "kernels.h"
#include "metadata.cuh"

namespace cdb {

constexpr int HN_THREADS = 128;
constexpr uint32_t HN_EMPTY = 0xFFFFFFFFu;
constexpr uint32_t HN_ROOT_ID = 0xFFFFFFFFu;
constexpr uint32_t HN_QUERY_ID = 0xFFFFFFFEu;  // hnsw/mod.rs:398
constexpr uint32_t HN_MAX_TAKE = 64;            // slots examined per pop (<= shortlist_size, config.toml:32)

struct HnSmem {
    uint8_t *qs;        // [row_pitch] the query / new vector, stored layout
    uint64_t *qkeys;    // [2][EFP] candidate queue (double buffered), sorted best first
    uint64_t *rkeys;    // [EFP] popped entries (results)
    uint64_t *nkeys;    // [64] new entries + [64] sorted copy
    uint64_t *fs;       // [64] PerformantFixedSet buckets
    uint32_t *qnodes, *rnodes, *nnodes;
    uint32_t EFP;
    uint8_t *stage;     // [stage_rows][stage_pitch] neighbour rows of the current pop, staged by the whole CTA
    uint32_t stage_pitch, stage_rows;
};
struct HnShared {
    uint32_t qlen, cur, visited, rlen, ncand, err, entry;
    uint32_t accmask[2];   // accepted slots of the current pop (slot order is kept: the reference scores them in that order)
    uint32_t err_first;    // (position << 8 | flag) of the first failing evaluation of the current pop
    uint32_t bitkey[HN_MAX_TAKE];
    uint32_t nrow[HN_MAX_TAKE];   // vector rows of the accepted neighbours
};
// metadata-filtered search (cosine.rs:34-102): per-node replica ids / metadata rows of the level and the query-side metadata
struct HnMdCtx {
    const uint32_t *node_id;   // [cnt] ProbNode::get_id()
    const uint32_t *node_md;   // [cnt] row of the metadata table, HN_EMPTY = prop_metadata None
    const int32_t *md_bits;    // [n_md][M]
    const float *md_mags;      // [n_md]
    uint32_t M;
    const int32_t *q_bits;     // query-side Metadata.mbits (shared memory), nullptr = None
    float q_mag;
    bool keep_fs;              // keep the fixed set of the previous traversal of this level (vector_store.rs:266-291)
    bool q_has_id;             // fvec_data.id: None for queries, Some(prop_value.id) while indexing (vector_store.rs:812, 1131-1135)
    uint32_t q_id;
};
struct HnScoreCtx {
    const uint8_t *rows;
    uint32_t row_pitch;
    const float *mags;
    uint32_t dim;
    int st, metric;
    uint32_t root_row;
};

__host__ __device__ inline uint32_t hn_efp(uint32_t ef) {
    uint32_t p = 1;
    while (p < ef) p <<= 1;
    return p < 128 ? 128u : p;
}
// Staging buffer: per pop only a handful of neighbours are scored, each by ONE thread (the reference arithmetic is a
// sequential chain per pair), so per-thread row reads would expose one memory round trip per 128 bytes.  Instead all
// threads of the CTA copy the rows of a group of neighbours into shared memory with 16-byte cp.async (one round trip for the
// whole group) and the scoring threads read shared memory.  Row pitch + 16 bytes keeps the threads on different banks.
constexpr uint32_t HN_STAGE_BYTES = 18 * 1024;
__host__ __device__ inline uint32_t hn_stage_pitch(uint32_t row_pitch) { return round_up(row_pitch, 16) + 16; }
__host__ __device__ inline uint32_t hn_stage_rows(uint32_t row_pitch) {
    const uint32_t r = HN_STAGE_BYTES / hn_stage_pitch(row_pitch);
    return r > HN_MAX_TAKE ? HN_MAX_TAKE : (r ? r : 1u);
}
__host__ __device__ inline size_t hn_base_bytes(uint32_t row_pitch, uint32_t ef) {
    const uint32_t efp = hn_efp(ef);
    return round_up(row_pitch, 16) + (size_t)(3 * efp + 2 * HN_MAX_TAKE + 64) * 8 + (size_t)(3 * efp + 2 * HN_MAX_TAKE) * 4 + 64;
}
__host__ __device__ inline size_t hn_smem_bytes(uint32_t row_pitch, uint32_t ef) {
    return (hn_base_bytes(row_pitch, ef) + 15) / 16 * 16 + (size_t)hn_stage_rows(row_pitch) * hn_stage_pitch(row_pitch);
}
__device__ __forceinline__ void hn_cp_async16(void *smem_dst, const void *gsrc) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(__cvta_generic_to_global(gsrc)) : "memory");
}
__device__ __forceinline__ void hn_cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ uint32_t hw_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
// TMA bulk copy (UBLKCP): `bytes` contiguous bytes global -> shared, completion counted on the mbarrier.  One instruction
// per row, issued by one lane: no per-lane address arithmetic, no LSU slots (the CTA traversal issues 96 cp.async per f16 x 768 row).
__device__ __forceinline__ void hw_bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void hw_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void hw_mbar_expect(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void hw_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
__device__ inline HnSmem hn_carve(uint8_t *smem, uint32_t row_pitch, uint32_t ef) {
    HnSmem m;
    m.EFP = hn_efp(ef);
    m.qs = smem;
    m.qkeys = reinterpret_cast<uint64_t *>(smem + round_up(row_pitch, 16));
    m.rkeys = m.qkeys + 2 * m.EFP;
    m.nkeys = m.rkeys + m.EFP;
    m.fs = m.nkeys + 2 * HN_MAX_TAKE;
    m.qnodes = reinterpret_cast<uint32_t *>(m.fs + 64);
    m.rnodes = m.qnodes + 2 * m.EFP;
    m.nnodes = m.rnodes + m.EFP;
    m.stage = smem + (hn_base_bytes(row_pitch, ef) + 15) / 16 * 16;
    m.stage_pitch = hn_stage_pitch(row_pitch);
    m.stage_rows = hn_stage_rows(row_pitch);
    return m;
}
__device__ __forceinline__ uint32_t hn_id(uint32_t root_row, uint32_t row) { return row == root_row ? HN_ROOT_ID : row; }

// metadata search (hnsw_md.cu, hnsw_warp.cu): a pseudo node's results carry no vector row
__device__ __forceinline__ bool hnm_is_pseudo(const HnswMdArgs &a, int level, uint32_t node) {
    const uint32_t mrow = a.node_md[level][node];
    if (mrow == HN_EMPTY || a.md_mags[mrow] == 0.0f) return false;
    const uint32_t id = a.node_id[level][node];
    return id >= MD_PSEUDO_ID_LO && id <= MD_PSEUDO_ID_HI;
}
// rows [*f0, *f1) of filter_dims for filtered query qi.  The offsets may come from device memory the host never read, so a
// range that is not off[q] <= off[q+1] <= n_filter_rows with at most HN_MAX_FILTERS rows fails the query (false, empty range).
constexpr uint32_t HN_MAX_FILTERS = 4096;
__device__ __forceinline__ bool hnm_filter_rows(const HnswMdArgs &a, uint32_t qi, uint32_t *f0, uint32_t *f1) {
    const uint32_t lo = a.filter_offsets[qi], hi = a.filter_offsets[qi + 1];
    const bool ok = lo <= hi && hi <= a.n_filter_rows && hi - lo <= HN_MAX_FILTERS;
    *f0 = ok ? lo : 0u;
    *f1 = ok ? hi : 0u;
    return ok;
}

// bitonic sort (descending) of n keys with a payload, padded to P (power of two) with zeros
__device__ inline void hn_sort_desc(uint64_t *keys, uint32_t *vals, uint32_t n, uint32_t P) {
    for (uint32_t i = n + threadIdx.x; i < P; i += blockDim.x) { keys[i] = 0ull; vals[i] = 0; }
    __syncthreads();
    for (uint32_t size = 2; size <= P; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t x = keys[lo], y = keys[hi];
                if ((x < y) == desc) {
                    keys[lo] = y; keys[hi] = x;
                    const uint32_t v = vals[lo]; vals[lo] = vals[hi]; vals[hi] = v;
                }
            }
            __syncthreads();
        }
    }
}

// One level.  On return (sh.err == 0) rkeys/rnodes[0..sh.rlen) hold every popped entry sorted best first
// (the caller truncates to 100 / 64).  All threads of the CTA must call it.  `self_id` is pre-inserted into the
// fixed set (the query id while searching, the new node's id while indexing: vector_store.rs:271, 807).
// score node `local` of the level against the query (reference arithmetic); *id = the id the fixed set / keys use
__device__ __forceinline__ int hn_score_node(const uint32_t *__restrict__ node_row, uint32_t local, const HnScoreCtx &sc, const HnSmem &m,
                                             float qmag, uint32_t pp, const HnMdCtx *md, float *d, uint32_t *id,
                                             const uint8_t *staged = nullptr) {
    const uint32_t row = node_row[local];
    const uint8_t *code = staged ? staged : sc.rows + (size_t)row * sc.row_pitch;
    if (!md) {
        *id = hn_id(sc.root_row, row);
        return pair_distance(sc.metric, sc.st, sc.dim, m.qs, qmag, pp, code, sc.mags[row], pp, d);
    }
    *id = md->node_id[local];
    const uint32_t mrow = md->node_md[local];
    const MdSide x{m.qs, qmag, pp, md->q_has_id, md->q_id, md->q_bits, md->q_mag};
    const MdSide y{code, sc.mags[row], pp, true, *id, mrow == HN_EMPTY ? nullptr : md->md_bits + (size_t)mrow * md->M,
                   mrow == HN_EMPTY ? 0.0f : md->md_mags[mrow]};
    return md_pair_distance(sc.metric, sc.st, sc.dim, md->M, x, y, d);
}

__device__ inline void hn_traverse_level(const uint32_t *__restrict__ node_row, const uint32_t *__restrict__ adj, uint32_t nb,
                                         uint32_t take, const HnScoreCtx &sc, const HnSmem &m, HnShared &sh, float qmag,
                                         uint32_t self_id, uint32_t ef, unsigned long long &evals, unsigned long long &pops,
                                         const HnMdCtx *md = nullptr, bool seed_self = true) {
    // seed_self = false: nothing is pre-inserted into the fixed set (delete_embedding, vector_store.rs:1231-1235)
    const int tid = threadIdx.x;
    const uint32_t pp = plane_pitch(sc.dim);
    const uint32_t EFP = m.EFP;
    const bool keep_fs = md && md->keep_fs;
    if (tid < 64 && !keep_fs) m.fs[tid] = 0ull;
    __syncthreads();
    if (tid == 0) {
        const uint32_t mask = nb - 1u;
        if (seed_self) m.fs[(self_id >> 6) & mask] |= 1ull << (self_id & 0x3f);
        const uint32_t entry = sh.entry;
        float d = 0.f;
        uint32_t eid;
        const int rc = hn_score_node(node_row, entry, sc, m, qmag, pp, md, &d, &eid);
        evals++;
        if (rc != CDB_OK) sh.err = md_err_flag(rc);
        m.fs[(eid >> 6) & mask] |= 1ull << (eid & 0x3f);
        m.qkeys[0] = make_key64(order_key(sc.metric, __float_as_uint(d)), eid);
        m.qnodes[0] = entry;
        sh.qlen = 1; sh.cur = 0; sh.visited = 0; sh.rlen = 0;
    }
    __syncthreads();
    if (sh.err) return;

    while (true) {
        const uint32_t qlen = sh.qlen, cur = sh.cur, visited = sh.visited;
        if (qlen == 0 || visited >= ef) break;
        uint64_t *Q = m.qkeys + cur * EFP;
        uint32_t *QN = m.qnodes + cur * EFP;
        // ---- pop (one thread), then the walk through the lossy fixed set for all slots at once.
        // The reference tests and inserts slot by slot: a slot is scored iff its bit is not yet set AND no
        // earlier non-empty slot of this pop maps to the same bit (that one either set it or found it set).
        const uint32_t bn = QN[0];
        if (tid == 0) {
            m.rkeys[sh.rlen] = Q[0]; m.rnodes[sh.rlen] = bn; sh.rlen++;
            pops++;
            sh.ncand = 0;
        }
        uint32_t my_nbl = HN_EMPTY, my_bitkey = 0xFFFFFFFFu;
        if (tid == 0) sh.err_first = 0xFFFFFFFFu;
        if ((uint32_t)tid < take) {
            my_nbl = adj[(size_t)bn * nb + tid];
            if (my_nbl != HN_EMPTY) {
                const uint32_t id = md ? md->node_id[my_nbl] : hn_id(sc.root_row, node_row[my_nbl]);
                my_bitkey = (((id >> 6) & (nb - 1u)) << 6) | (id & 0x3f);
            }
            sh.bitkey[tid] = my_bitkey;
        }
        __syncthreads();
        bool accept = false;
        if (my_bitkey != 0xFFFFFFFFu) {
            accept = ((m.fs[my_bitkey >> 6] >> (my_bitkey & 0x3f)) & 1ull) == 0;
            for (int s2 = 0; s2 < tid && accept; ++s2) accept = sh.bitkey[s2] != my_bitkey;
        }
        const uint32_t ball = __ballot_sync(0xFFFFFFFFu, accept);   // HN_MAX_TAKE = 64: warps 0 and 1 hold every slot
        if ((tid & 31) == 0 && tid < 64) sh.accmask[tid >> 5] = ball;
        __syncthreads();  // every thread has read the old fixed set
        if (accept) {
            atomicOr(reinterpret_cast<unsigned long long *>(&m.fs[my_bitkey >> 6]), 1ull << (my_bitkey & 0x3f));
            const uint32_t rank = (tid < 32 ? 0u : (uint32_t)__popc(sh.accmask[0])) + (uint32_t)__popc(ball & ((1u << (tid & 31)) - 1u));
            m.nnodes[rank] = my_nbl;   // compacted in slot order
        }
        if (tid == 0) sh.ncand = (uint32_t)(__popc(sh.accmask[0]) + __popc(sh.accmask[1]));
        __syncthreads();
        const uint32_t nc = sh.ncand;
        // ---- score the new neighbours, one thread each, reference arithmetic, rows staged through shared memory
        if ((uint32_t)tid < nc) sh.nrow[tid] = node_row[m.nnodes[tid]];
        __syncthreads();
        {
            const uint32_t cpr = sc.row_pitch >> 4;   // 16-byte chunks per stored row
            for (uint32_t g0 = 0; g0 < nc; g0 += m.stage_rows) {
                const uint32_t gn = min(m.stage_rows, nc - g0);
                for (uint32_t c = tid; c < gn * cpr; c += HN_THREADS) {
                    const uint32_t r = c / cpr, o = c - r * cpr;
                    hn_cp_async16(m.stage + (size_t)r * m.stage_pitch + (size_t)o * 16,
                                  sc.rows + (size_t)sh.nrow[g0 + r] * sc.row_pitch + (size_t)o * 16);
                }
                hn_cp_async_wait_all();
                __syncthreads();
                if ((uint32_t)tid < gn) {
                    const uint32_t pos = g0 + tid;
                    float d = 0.f;
                    uint32_t nid;
                    const int rc = hn_score_node(node_row, m.nnodes[pos], sc, m, qmag, pp, md, &d, &nid, m.stage + (size_t)tid * m.stage_pitch);
                    if (rc != CDB_OK) atomicMin(&sh.err_first, (pos << 8) | md_err_flag(rc));   // the reference stops at the first Err
                    m.nkeys[pos] = make_key64(order_key(sc.metric, __float_as_uint(d)), nid);
                }
                __syncthreads();   // the stage is reused by the next group
            }
        }
        if (tid == 0) evals += nc;
        if (sh.err_first != 0xFFFFFFFFu) {
            if (tid == 0) sh.err = sh.err_first & 0xFFu;
            __syncthreads();
            return;
        }
        // ---- sort the new entries (rank sort, nc <= 64) into nkeys[64..], nnodes[64..]
        if ((uint32_t)tid < nc) {
            const uint64_t k = m.nkeys[tid];
            uint32_t r = 0;
            for (uint32_t j = 0; j < nc; ++j) r += m.nkeys[j] > k;
            m.nkeys[HN_MAX_TAKE + r] = k;
            m.nnodes[HN_MAX_TAKE + r] = m.nnodes[tid];
        }
        __syncthreads();
        // ---- merge the old queue (minus the popped head) with the new entries, keep what can still be popped
        {
            const uint64_t *NK = m.nkeys + HN_MAX_TAKE;
            const uint32_t *NN = m.nnodes + HN_MAX_TAKE;
            const uint32_t oldn = qlen - 1;
            const uint32_t cap = min(ef - (visited + 1), EFP);  // pops still to come
            uint64_t *D = m.qkeys + (cur ^ 1) * EFP;
            uint32_t *DN = m.qnodes + (cur ^ 1) * EFP;
            for (uint32_t i = tid; i < oldn; i += HN_THREADS) {
                const uint64_t k = Q[1 + i];
                uint32_t lo = 0, hi = nc;  // number of new entries better than k
                while (lo < hi) { const uint32_t md = (lo + hi) >> 1; if (NK[md] > k) lo = md + 1; else hi = md; }
                const uint32_t pos = i + lo;
                if (pos < cap) { D[pos] = k; DN[pos] = QN[1 + i]; }
            }
            for (uint32_t j = tid; j < nc; j += HN_THREADS) {
                const uint64_t k = NK[j];
                uint32_t lo = 0, hi = oldn;  // number of old entries better than k
                while (lo < hi) { const uint32_t md = (lo + hi) >> 1; if (Q[1 + md] > k) lo = md + 1; else hi = md; }
                const uint32_t pos = j + lo;
                if (pos < cap) { D[pos] = k; DN[pos] = NN[j]; }
            }
            __syncthreads();
            if (tid == 0) { sh.qlen = min(oldn + nc, cap); sh.cur = cur ^ 1; sh.visited = visited + 1; }
        }
        __syncthreads();
    }
    __syncthreads();
    const uint32_t rlen = sh.rlen;
    uint32_t P = 1;
    while (P < rlen) P <<= 1;
    hn_sort_desc(m.rkeys, m.rnodes, rlen, P);
}

}  // namespace cdb
