// hnsw_warp.cu -- batched HNSW search, ONE WARP PER QUERY (S1, CDB_MODE_HNSW on graphs without metadata):
//   ann_search              src/vector_store.rs:256-402
//   traverse_find_nearest   src/vector_store.rs:1112-1204
//   PerformantFixedSet      src/models/fixedset.rs:2-29
//
// Why a warp.  A traversal is a chain of dependent pops; per pop only ~6 neighbours survive the fixed set, and each of
// them is scored by ONE thread because the reference arithmetic is a sequential chain per pair (dot_product_f16 is a
// left fold: 768 dependent adds).  The round-1 kernel gave every query a 128-thread CTA: three of its four warps waited
// at 9 block barriers per pop while one warp ran the chains (ncu: 63 % of warp samples parked at the barrier, 0.27 IPC on
// the scoring warp).  Here the 32 lanes of one warp ARE the neighbour slots (two slots per lane cover the <= 64 slots a
// pop examines), every hand-over is a __syncwarp / ballot / match, and the SM's four schedulers each see ~2 independent
// queries whose chains interleave.  Queue, results, fixed set and the staged neighbour rows live in the warp's slice of
// shared memory (~24 KB at ef = 128, f16 x 768), so 7-9 queries are resident per SM -- all 1024 queries of a batch at once.
//
// Parity.  Pop order, fixed-set walk (slot order, aliasing ids included), first-Err rule, the (score, id) key and the
// per-level bookkeeping are those of hn_traverse_level (hnsw_traverse.cuh), which the builder and the metadata search keep
// using; tests/test_gpu_hnsw.py checks ids, scores, counts, error flags AND the evaluation / pop counts against the oracle.
//
// f16 chain.  dot_product_f16 = sum_i f32(x_i) * f32(y_i), sequential, no FMA in the reference.  The product of two
// halfs is exact in f32 (11 + 11 significand bits, exponent range far inside f32), so fma(x, y, s) rounds exactly once
// at the same place as s + (x * y): one fused multiply-add per element instead of FMUL + FADD, bit-identical.  The 16-bit
// operands are widened exactly from the packed registers (scorers.cuh, widen16), so no f32 query copy is needed.
#include <cstdlib>

#include "hnsw_traverse.cuh"

namespace cdb {

constexpr uint32_t HW_FINAL_LEN = 100;          // vector_store.rs:1194
// staged neighbour rows per group, sized so that 7 warps (queries) per SM still fit in shared memory at D = 768:
constexpr uint32_t HW_STAGE_BYTES = 18700;      // 12 rows of f16 x 768, 6 of f32 x 768
constexpr uint32_t HW_STAGE_BYTES_SPEC = 20200; // speculative form (score cache + work list added): 13 rows of f16 x 768
constexpr uint32_t HW_CACHE = 256;              // speculative form: direct-mapped (node -> score key) cache entries per query
constexpr int HW_NSRC = 3;                      // speculative form: upcoming heads examined per chain phase
constexpr uint32_t HW_WORK = HN_MAX_TAKE + 32;  // speculative form: rows to score in one pop (misses of the head + fill)
// clock64 sums per query (lane 0): [0] pop + adjacency (+ node_row) loads, [1] fixed-set walk + compaction + prefetches,
// [2] issue of the row copies, [3] wait for the rows, [4] distance chains, [5] queue merge, [6] end-of-level result sort,
// [7] whole levels, [8] pops
// speculative form: [9] cache look-ups + choice of speculative rows, [10] chain phases, [11] speculative evaluations
constexpr int HW_PROF_SLOTS = 12;

struct HwCarve {
    uint32_t EFP, stage_pitch, stage_rows;
    uint32_t off_q32, off_qkeys, off_rkeys, off_nkeys, off_fs, off_qnodes, off_rnodes, off_nnodes, off_nrow, off_bar, off_stage, total;
    uint32_t off_cache, off_work, off_sadj;   // speculative form only
};

__host__ __device__ inline HwCarve hw_carve(uint32_t row_pitch, uint32_t dim, uint32_t ef, bool f16fast, bool spec = false) {
    HwCarve c;
    c.EFP = hn_efp(ef);
    c.stage_pitch = round_up(row_pitch, 16) + 16;   // + 16 bytes: the lanes' rows start on different banks
    uint32_t r = (spec ? HW_STAGE_BYTES_SPEC : HW_STAGE_BYTES) / c.stage_pitch;
    c.stage_rows = r > 32 ? 32 : (r ? r : 1u);      // one lane scores one staged row
    uint32_t o = round_up(row_pitch, 16);
    c.off_q32 = o;            // (no f32 copy of the query: the chain widens the f16 / bf16 code directly)
    c.off_qkeys = o;          o += 2 * c.EFP * 8;
    c.off_rkeys = o;          o += c.EFP * 8;
    c.off_nkeys = o;          o += HN_MAX_TAKE * 8;
    c.off_bar = o;            o += 8;
    c.off_fs = o;             o += 128 * 4;
    c.off_qnodes = o;         o += 2 * c.EFP * 4;
    c.off_rnodes = o;         o += c.EFP * 4;
    c.off_nnodes = o;         o += HN_MAX_TAKE * 4;
    c.off_nrow = o;           o += HN_MAX_TAKE * 4;
    c.off_cache = c.off_work = c.off_sadj = 0;
    if (spec) {
        o = round_up(o, 8);
        c.off_cache = o;      o += HW_CACHE * 8;
        c.off_work = o;       o += 3 * HW_WORK * 4;
        c.off_sadj = o;       o += HW_NSRC * HN_MAX_TAKE * 4;
    }
    c.off_stage = round_up(o, 16);
    c.total = c.off_stage + c.stage_rows * c.stage_pitch;
    return c;
}

struct HwSmem {
    uint8_t *qs;
    float *q32;
    uint64_t *qkeys, *rkeys, *nkeys;
    uint32_t *fs;            // PerformantFixedSet as 128 x 32-bit words: bucket b = words 2b, 2b+1 (native 32-bit shared atomics)
    uint32_t *qnodes, *rnodes, *nnodes, *nrow;
    uint64_t *cache;         // speculative form: (node << 32 | score order key), tag 0xFFFFFFFF = empty
    uint32_t *wnode, *wrow, *wdst;
    uint32_t *sadj;          // speculative form: adjacency slots of the next heads, [HW_NSRC][64], filled by cp.async
    uint8_t *stage;
    uint32_t bar;            // shared-space address of the warp's mbarrier (row copies complete on it)
    uint32_t EFP, stage_pitch, stage_rows;
};

__device__ __forceinline__ void hw_prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ uint32_t hw_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
// TMA bulk copy (UBLKCP): `bytes` contiguous bytes global -> shared, completion counted on the mbarrier.  One instruction
// per row, issued by one lane: no per-lane address arithmetic, no LSU slots (the round-1 kernel issued 96 cp.async per row).
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

// sum_i f32(q_i) * f32(row_i), sequential: both 16-bit operands widened exactly, then one FFMA rounding a*b + c once in
// f32 -- (the product of two halfs / two bf16 values being exact in f32) the same result as the reference's
// multiply-then-add.  No f32 copy of the query: 8 FFMA + their conversions + 2 LDS.128 per 8 elements.
// The chain is latency bound (one dependent FMA per element), so the shared-memory operands of the NEXT 16 elements are
// loaded before the current 16 FMAs issue (explicit double buffering: ptxas does not pipeline this loop itself).
template <int FAST>
__device__ __forceinline__ float hw_fhfma(float s, uint32_t q, uint32_t r, bool hi) {
    return FAST == 1 ? fhfma16<false>(s, q, r, hi) : fhfma16<true>(s, q, r, hi);
}
template <int FAST>
__device__ __forceinline__ float hw_chain8(float s, const uint4 &q, const uint4 &r) {
    s = hw_fhfma<FAST>(s, q.x, r.x, false); s = hw_fhfma<FAST>(s, q.x, r.x, true);
    s = hw_fhfma<FAST>(s, q.y, r.y, false); s = hw_fhfma<FAST>(s, q.y, r.y, true);
    s = hw_fhfma<FAST>(s, q.z, r.z, false); s = hw_fhfma<FAST>(s, q.z, r.z, true);
    s = hw_fhfma<FAST>(s, q.w, r.w, false); s = hw_fhfma<FAST>(s, q.w, r.w, true);
    return s;
}
struct HwBlk16 { uint4 r0, r1, q0, q1; };
__device__ __forceinline__ HwBlk16 hw_ld16(const uint8_t *__restrict__ q, const uint8_t *__restrict__ row, uint32_t i) {
    HwBlk16 b;
    b.r0 = *reinterpret_cast<const uint4 *>(row + 2 * i);
    b.r1 = *reinterpret_cast<const uint4 *>(row + 2 * i + 16);
    b.q0 = *reinterpret_cast<const uint4 *>(q + 2 * i);
    b.q1 = *reinterpret_cast<const uint4 *>(q + 2 * i + 16);
    return b;
}
// q: the query's f16 / bf16 code in shared memory (16-byte aligned, like the staged row)
template <int FAST>
__device__ __forceinline__ float hw_dot16(const uint8_t *__restrict__ q, const uint8_t *__restrict__ row, uint32_t n) {
    float s = 0.0f;
    const uint32_t n16 = n & ~15u;
    uint32_t i = 0;
    if (n16) {
        HwBlk16 cur = hw_ld16(q, row, 0);
        for (; i + 16 < n16; i += 16) {
            const HwBlk16 nxt = hw_ld16(q, row, i + 16);
            s = hw_chain8<FAST>(s, cur.q0, cur.r0);
            s = hw_chain8<FAST>(s, cur.q1, cur.r1);
            cur = nxt;
        }
        s = hw_chain8<FAST>(s, cur.q0, cur.r0);
        s = hw_chain8<FAST>(s, cur.q1, cur.r1);
        i = n16;
    }
    if (i + 8 <= n) {
        s = hw_chain8<FAST>(s, *reinterpret_cast<const uint4 *>(q + 2 * i), *reinterpret_cast<const uint4 *>(row + 2 * i));
        i += 8;
    }
    for (; i < n; ++i) {
        const uint32_t qa = reinterpret_cast<const uint16_t *>(q)[i], ra = reinterpret_cast<const uint16_t *>(row)[i];
        s = hw_fhfma<FAST>(s, qa, ra, false);
    }
    return s;
}

// warp bitonic sort, descending, n keys padded to P (power of two) with zeros
__device__ inline void hw_sort_desc(uint64_t *keys, uint32_t *vals, uint32_t n, uint32_t P, int lane) {
    for (uint32_t i = n + lane; i < P; i += 32) { keys[i] = 0ull; vals[i] = 0; }
    __syncwarp();
    for (uint32_t size = 2; size <= P; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = lane; t < P / 2; t += 32) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t x = keys[lo], y = keys[hi];
                if ((x < y) == desc) {
                    keys[lo] = y; keys[hi] = x;
                    const uint32_t v = vals[lo]; vals[lo] = vals[hi]; vals[hi] = v;
                }
            }
            __syncwarp();
        }
    }
}

struct HwState {
    uint32_t err, rlen, bar_phase;
    unsigned long long evals, pops;
    long long prof[HW_PROF_SLOTS];
};

// Score the compacted neighbours nnodes/nrow[first .. first+n) into nkeys (slot order kept).  Rows are staged through
// shared memory (one TMA bulk copy per row, all in flight together: one memory round trip per group), then one lane per
// row runs the reference chain.  Returns the (position << 8 | flag) of the first failing evaluation, 0xFFFFFFFF if none.
template <int FAST, bool PROF>
__device__ __forceinline__ uint32_t hw_score_group(const HnScoreCtx &sc, const HwSmem &m, float qmag, uint32_t pp, uint32_t first,
                                                   uint32_t n, int lane, HwState &st) {
    uint32_t err_first = 0xFFFFFFFFu;
    for (uint32_t g0 = 0; g0 < n; g0 += m.stage_rows) {
        const uint32_t gn = min(m.stage_rows, n - g0);
        long long ts = 0, ti = 0, tw = 0;
        if (PROF) ts = clock64();
        uint32_t row = 0;
        float rmag = 0.0f;
        // (a copy may complete before the expect_tx is posted: the phase cannot end before lane 0's arrive)
        if (lane == 0) hw_mbar_expect(m.bar, gn * sc.row_pitch);
        if ((uint32_t)lane < gn) {
            row = m.nrow[first + g0 + lane];
            hw_bulk_g2s(hw_smem_u32(m.stage + (size_t)lane * m.stage_pitch), sc.rows + (size_t)row * sc.row_pitch, sc.row_pitch, m.bar);
            rmag = sc.mags[row];   // in flight together with the rows
        }
        if (PROF) ti = clock64();
        hw_mbar_wait(m.bar, st.bar_phase);
        st.bar_phase ^= 1u;
        if (PROF) tw = clock64();
        int rc = CDB_OK;
        if ((uint32_t)lane < gn) {
            const uint32_t pos = first + g0 + lane;
            const uint8_t *code = m.stage + (size_t)lane * m.stage_pitch;
            float d = 0.0f;
            if (FAST) {
                const float dot = hw_dot16<FAST>(m.qs, code, sc.dim);
                if (sc.metric == CDB_METRIC_COSINE) {
                    const float denom = __fmul_rn(qmag, rmag);
                    if (denom == 0.0f) rc = CDB_CALCULATION_ERROR;   // cosine.rs:230-231
                    else d = canon_nan(__fdiv_rn(dot, denom));
                } else {
                    d = dot;
                }
            } else {
                rc = pair_distance(sc.metric, sc.st, sc.dim, m.qs, qmag, pp, code, rmag, pp, &d);
            }
            m.nkeys[pos] = make_key64(order_key(sc.metric, __float_as_uint(d)), hn_id(sc.root_row, row));
        }
        const uint32_t bad = __ballot_sync(0xFFFFFFFFu, rc != CDB_OK);
        if (bad && err_first == 0xFFFFFFFFu) {   // the reference stops at the first Err (slot order)
            const int src_lane = __ffs(bad) - 1;
            const int flag = __shfl_sync(0xFFFFFFFFu, (int)md_err_flag(rc), src_lane);
            err_first = ((first + g0 + (uint32_t)src_lane) << 8) | (uint32_t)flag;
        }
        __syncwarp();   // nkeys written; the stage is reused by the next group
        if (PROF) { const long long te = clock64(); st.prof[2] += ti - ts; st.prof[3] += tw - ti; st.prof[4] += te - tw; }
    }
    return err_first;
}

__device__ __forceinline__ uint32_t hw_cache_slot(uint32_t node) { return (node * 0x9E3779B1u) >> 24; }   // HW_CACHE = 256

// Speculative form: score the work list wnode/wrow[0 .. nt).  Entries [0, nm) are the head's neighbours whose score is not
// cached (slot order kept; the key goes to nkeys[wdst]); entries [nm, nt) are neighbours of upcoming heads that fill the
// otherwise idle lanes of the chain phase -- their score keys go to the cache (an evaluation that fails is simply not cached:
// the error belongs to the pop that commits it).  Same staging and the same chains as hw_score_group.
template <int FAST, bool PROF>
__device__ __forceinline__ uint32_t hw_score_work(const HnScoreCtx &sc, const HwSmem &m, float qmag, uint32_t pp, uint32_t nm,
                                                  uint32_t nt, int lane, HwState &st) {
    uint32_t err_first = 0xFFFFFFFFu;
    for (uint32_t g0 = 0; g0 < nt; g0 += m.stage_rows) {
        const uint32_t gn = min(m.stage_rows, nt - g0);
        long long ts = 0, ti = 0, tw = 0;
        if (PROF) ts = clock64();
        uint32_t row = 0;
        float rmag = 0.0f;
        if (lane == 0) hw_mbar_expect(m.bar, gn * sc.row_pitch);
        if ((uint32_t)lane < gn) {
            row = m.wrow[g0 + lane];
            hw_bulk_g2s(hw_smem_u32(m.stage + (size_t)lane * m.stage_pitch), sc.rows + (size_t)row * sc.row_pitch, sc.row_pitch, m.bar);
            rmag = sc.mags[row];
        }
        if (PROF) ti = clock64();
        hw_mbar_wait(m.bar, st.bar_phase);
        st.bar_phase ^= 1u;
        if (PROF) tw = clock64();
        int rc = CDB_OK;
        const uint32_t idx = g0 + (uint32_t)lane;
        if ((uint32_t)lane < gn) {
            const uint8_t *code = m.stage + (size_t)lane * m.stage_pitch;
            float d = 0.0f;
            if (FAST) {
                const float dot = hw_dot16<FAST>(m.qs, code, sc.dim);
                if (sc.metric == CDB_METRIC_COSINE) {
                    const float denom = __fmul_rn(qmag, rmag);
                    if (denom == 0.0f) rc = CDB_CALCULATION_ERROR;   // cosine.rs:230-231
                    else d = canon_nan(__fdiv_rn(dot, denom));
                } else {
                    d = dot;
                }
            } else {
                rc = pair_distance(sc.metric, sc.st, sc.dim, m.qs, qmag, pp, code, rmag, pp, &d);
            }
            const uint32_t okey = order_key(sc.metric, __float_as_uint(d));
            if (idx < nm) m.nkeys[m.wdst[idx]] = make_key64(okey, hn_id(sc.root_row, row));
            else if (rc == CDB_OK) { const uint32_t nd = m.wnode[idx]; m.cache[hw_cache_slot(nd)] = ((uint64_t)nd << 32) | okey; }
        }
        const uint32_t bad = __ballot_sync(0xFFFFFFFFu, rc != CDB_OK && idx < nm);
        if (bad && err_first == 0xFFFFFFFFu) {   // the reference stops at the first Err (slot order)
            const int src_lane = __ffs(bad) - 1;
            const int flag = __shfl_sync(0xFFFFFFFFu, (int)md_err_flag(rc), src_lane);
            err_first = ((g0 + (uint32_t)src_lane) << 8) | (uint32_t)flag;
        }
        __syncwarp();
        if (PROF) { const long long te = clock64(); st.prof[2] += ti - ts; st.prof[3] += tw - ti; st.prof[4] += te - tw; st.prof[10] += 1; }
    }
    return err_first;
}

// One level (traverse_find_nearest).  All 32 lanes call it with warp-uniform arguments.  On return (st.err == 0)
// rkeys/rnodes[0..st.rlen) hold every popped entry sorted best first.
template <int FAST, bool PROF>
__device__ void hw_traverse_level(const uint32_t *__restrict__ node_row /* null: identity */, const uint32_t *__restrict__ adj,
                                  uint32_t nb, uint32_t take, const HnScoreCtx &sc, const HwSmem &m, float qmag, uint32_t self_id,
                                  uint32_t ef, uint32_t entry, HwState &st, int lane, uint32_t flags) {
    const uint32_t pp = plane_pitch(sc.dim);
    const bool f_preload = (flags & CDB_HNSW_F_PRELOAD) != 0, f_atomfs = (flags & CDB_HNSW_F_ATOMFS) != 0;
    const bool f_pool = (flags & CDB_HNSW_F_POOL) != 0;
    const bool f_spec = (flags & CDB_HNSW_F_SPEC) != 0 && !f_pool;
    const uint32_t EFP = m.EFP;
    const uint32_t CAPQ = 2 * EFP;      // pool form: both queue buffers are one unsorted pool
    const uint32_t bmask = nb - 1u;
    const uint32_t lt = (1u << lane) - 1u;
    long long t0 = 0;
    if (PROF) t0 = clock64();
#pragma unroll
    for (int i = 0; i < 4; ++i) m.fs[lane + 32 * i] = 0u;
    if (f_spec)   // node indices are level-local: the score cache starts empty on every level
        for (uint32_t i = lane; i < HW_CACHE; i += 32) m.cache[i] = ~0ull;
    uint32_t sd0 = HN_EMPTY, sd1 = HN_EMPTY, sd2 = HN_EMPTY, sd3 = HN_EMPTY;   // queue entries whose neighbours are all cached
    if (lane == 0) { m.nnodes[0] = entry; m.nrow[0] = node_row ? node_row[entry] : entry; }
    __syncwarp();
    {
        const uint32_t e = hw_score_group<FAST, PROF>(sc, m, qmag, pp, 0, 1, lane, st);
        st.evals += 1;
        if (e != 0xFFFFFFFFu) { st.err = e & 0xFFu; return; }
        if (lane == 0) {
            const uint32_t eid = hn_id(sc.root_row, m.nrow[0]);
            const uint32_t b0 = (((self_id >> 6) & bmask) << 6) | (self_id & 0x3f), b1 = (((eid >> 6) & bmask) << 6) | (eid & 0x3f);
            m.fs[b0 >> 5] |= 1u << (b0 & 31);
            m.fs[b1 >> 5] |= 1u << (b1 & 31);
            m.qkeys[0] = m.nkeys[0];
            m.qnodes[0] = entry;
        }
        __syncwarp();
    }
    uint32_t qlen = 1, cur = 0, visited = 0, rlen = 0;
    // adjacency slots of the head, loaded one pop ahead (while the previous pop's queue merge runs)
    uint32_t pre_node = HN_EMPTY, pre_nbl[2] = {HN_EMPTY, HN_EMPTY};
    // POOL form (CDB_HNSW_F_POOL): the candidates are an UNSORTED pool in shared memory and the head is found by an
    // arg-max (8 slots per lane, two 32-bit REDUX) instead of keeping a sorted queue that every pop has to merge into.
    // The pop order is the same: the head is the best entry present, and an entry is only ever dropped when at least
    // (pops still to come) better entries exist, so it could never have been popped.
    uint64_t hkey = f_pool ? m.qkeys[0] : 0ull;
    uint32_t hnode = entry;
    bool have_head = true;
    if (f_pool) qlen = 0;
    while ((f_pool ? have_head : qlen > 0) && visited < ef) {
        uint64_t *Q = m.qkeys + cur * EFP;
        uint32_t *QN = m.qnodes + cur * EFP;
        long long t1 = 0, t2 = 0, t3 = 0, t4 = 0;
        if (PROF) t1 = clock64();
        // ---- pop
        const uint32_t bn = f_pool ? hnode : QN[0];
        if (lane == 0) { m.rkeys[rlen] = f_pool ? hkey : Q[0]; m.rnodes[rlen] = bn; }
        ++rlen;
        st.pops += 1;
        // ---- adjacency: slots lane and lane + 32; ids and fixed-set bit positions
        uint32_t nbl[2], row[2], bk[2];
        if (pre_node == bn) {
            nbl[0] = pre_nbl[0]; nbl[1] = pre_nbl[1];
        } else {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t slot = (uint32_t)lane + 32u * h;
                nbl[h] = slot < take ? __ldg(adj + (size_t)bn * nb + slot) : HN_EMPTY;
            }
        }
        // SPECULATIVE form (CDB_HNSW_F_SPEC): a pop scores ~4 rows, so ~28 lanes idle through a 768-step dependent chain.  The
        // next heads are already known (the sorted queue), a score is a pure function of (query, node), and the fixed set only
        // grows: whatever a later pop will score is among the neighbours of that head whose bit is clear NOW.  So the free
        // lanes of this pop's chain phase score those rows ahead of time into a small cache; the later pop walks its fixed
        // set exactly as before (same order, same insertions, same evals count) and takes the keys from the cache, and a pop
        // whose accepted neighbours are all cached has no chain phase at all.
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            row[h] = 0;
            bk[h] = 0x80000000u | ((uint32_t)lane + 32u * h);   // unique per slot: never matches another slot
            if (nbl[h] != HN_EMPTY) {
                row[h] = node_row ? __ldg(node_row + nbl[h]) : nbl[h];
                const uint32_t id = hn_id(sc.root_row, row[h]);
                bk[h] = (((id >> 6) & bmask) << 6) | (id & 0x3f);
            }
        }
        uint32_t ssrc[HW_NSRC];
#pragma unroll
        for (int sidx = 0; sidx < HW_NSRC; ++sidx) ssrc[sidx] = HN_EMPTY;
        if (f_spec) {
            // the next queue entries whose neighbours are not all cached yet (lanes 1..6 look at one entry each).  Their adjacency
            // slots are copied to shared memory with cp.async: no registers and no scoreboard are held across the fixed-set walk
            // (register loads issued here made the walk's own shared-memory waits stall on the same scoreboards), and the data is
            // there when the chain phase of this pop -- if it has one -- chooses its fill
            const uint32_t mine = (lane >= 1 && (uint32_t)lane < qlen && lane <= 2 * HW_NSRC) ? QN[lane] : HN_EMPTY;
            uint32_t pick = __ballot_sync(0xFFFFFFFFu, mine != HN_EMPTY && mine != sd0 && mine != sd1 && mine != sd2 && mine != sd3);
#pragma unroll
            for (int sidx = 0; sidx < HW_NSRC; ++sidx)
                if (pick) { ssrc[sidx] = __shfl_sync(0xFFFFFFFFu, mine, __ffs(pick) - 1); pick &= pick - 1; }
            asm volatile("cp.async.wait_all;" ::: "memory");   // copies of the previous pop (long finished)
#pragma unroll
            for (int sidx = 0; sidx < HW_NSRC; ++sidx)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t slot = (uint32_t)lane + 32u * h;
                    if (ssrc[sidx] != HN_EMPTY && slot < take)
                        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(hw_smem_u32(m.sadj + sidx * HN_MAX_TAKE + slot)),
                                     "l"(adj + (size_t)ssrc[sidx] * nb + slot) : "memory");
                }
        }
        if (PROF) t2 = clock64();
        // ---- the walk through the lossy fixed set, slot order: a slot is scored iff its bit is not yet set AND no
        // earlier non-empty slot of this pop maps to the same bit (that one either set it or found it set).
        // Candidates = valid slots whose bit is clear (typically ~6).  They all set their bit with an atomicOr; if every
        // candidate finds it clear no two of them alias (the common case) and all are accepted.  Otherwise (two
        // candidate slots of one pop on the same bit, ~0.4 % of the pops) the slot-order rule is applied explicitly.
        bool accept[2];
        uint32_t nc = 0;
        {
            const bool two = take > 32;   // levels >= 1 examine <= 32 slots (neighbors_count 32): the second half is skipped there
            bool clear[2];
            clear[0] = nbl[0] != HN_EMPTY && ((m.fs[bk[0] >> 5] >> (bk[0] & 31)) & 1u) == 0;
            clear[1] = two && nbl[1] != HN_EMPTY && ((m.fs[bk[1] >> 5] >> (bk[1] & 31)) & 1u) == 0;
            const uint32_t cand0 = __ballot_sync(0xFFFFFFFFu, clear[0]);
            const uint32_t cand1 = two ? __ballot_sync(0xFFFFFFFFu, clear[1]) : 0u;
            accept[0] = clear[0]; accept[1] = clear[1];
            bool resolve = true;   // apply the slot-order rule explicitly
            if (f_atomfs) {
                bool won0 = false, won1 = false;
                if (clear[0]) { const uint32_t bit = 1u << (bk[0] & 31); won0 = (atomicOr(&m.fs[bk[0] >> 5], bit) & bit) == 0; }
                if (clear[1]) { const uint32_t bit = 1u << (bk[1] & 31); won1 = (atomicOr(&m.fs[bk[1] >> 5], bit) & bit) == 0; }
                const uint32_t w0 = __ballot_sync(0xFFFFFFFFu, won0);
                const uint32_t w1 = two ? __ballot_sync(0xFFFFFFFFu, won1) : 0u;
                resolve = __popc(w0) + __popc(w1) != __popc(cand0) + __popc(cand1);
            }
            if (resolve) {
                for (uint32_t rest = cand0; rest; rest &= rest - 1) {   // ascending slot order
                    const int c = __ffs(rest) - 1;
                    const uint32_t cb = __shfl_sync(0xFFFFFFFFu, bk[0], c);
                    if (lane > c && cb == bk[0]) accept[0] = false;     // an earlier slot of this pop owns the bit
                    if (cb == bk[1]) accept[1] = false;
                }
                for (uint32_t rest = cand1; rest; rest &= rest - 1) {
                    const int c = __ffs(rest) - 1;
                    const uint32_t cb = __shfl_sync(0xFFFFFFFFu, bk[1], c);
                    if (lane > c && cb == bk[1]) accept[1] = false;
                }
                if (!f_atomfs) {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (accept[h]) atomicOr(&m.fs[bk[h] >> 5], 1u << (bk[h] & 31));
                }
            }
            // without a conflict the accepted slots are exactly the candidates: no further ballot needed
            const uint32_t ball0 = resolve ? __ballot_sync(0xFFFFFFFFu, accept[0]) : cand0;
            const uint32_t ball1 = resolve ? __ballot_sync(0xFFFFFFFFu, accept[1]) : cand1;
            const uint32_t n0 = (uint32_t)__popc(ball0);
            nc = n0 + (uint32_t)__popc(ball1);
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (accept[h]) {
                    const uint32_t pos = (h ? n0 : 0u) + (uint32_t)__popc((h ? ball1 : ball0) & lt);   // compacted in slot order
                    m.nnodes[pos] = nbl[h];
                    m.nrow[pos] = row[h];
                    // the next head is often one of these: pull their adjacency rows towards L2 while the chains run
                    const uint8_t *ap = reinterpret_cast<const uint8_t *>(adj + (size_t)nbl[h] * nb);
                    hw_prefetch_l2(ap);
                    if (nb > 32) hw_prefetch_l2(ap + 128);
                }
            __syncwarp();   // compaction visible to the scoring
        }
        if (PROF) t3 = clock64();
        // ---- score the new neighbours
        uint32_t e = 0xFFFFFFFFu;
        if (f_spec) {
            // keys of accepted neighbours that were scored ahead of time; the others form the work list
            bool miss[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t pos = (uint32_t)lane + 32u * h;
                miss[h] = false;
                if (pos < nc) {
                    const uint32_t nd = m.nnodes[pos];
                    const uint64_t ce = m.cache[hw_cache_slot(nd)];
                    if ((uint32_t)(ce >> 32) == nd) m.nkeys[pos] = make_key64((uint32_t)ce, hn_id(sc.root_row, m.nrow[pos]));
                    else miss[h] = true;
                }
            }
            const uint32_t mb0 = __ballot_sync(0xFFFFFFFFu, miss[0]);
            const uint32_t mb1 = nc > 32 ? __ballot_sync(0xFFFFFFFFu, miss[1]) : 0u;
            const uint32_t nm0 = (uint32_t)__popc(mb0), nm = nm0 + (uint32_t)__popc(mb1);
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (miss[h]) {
                    const uint32_t pos = (uint32_t)lane + 32u * h;
                    const uint32_t w = (h ? nm0 : 0u) + (uint32_t)__popc((h ? mb1 : mb0) & lt);
                    m.wnode[w] = m.nnodes[pos]; m.wrow[w] = m.nrow[pos]; m.wdst[w] = pos;
                }
            uint32_t nt = nm;
            if (nm > 0 && nm < m.stage_rows) {
                asm volatile("cp.async.wait_all;" ::: "memory");   // every lane reads back exactly the slots it copied
                // one chain phase is due anyway: fill its free lanes with the uncached, not yet visited neighbours of the next heads
#pragma unroll
                for (int sidx = 0; sidx < HW_NSRC; ++sidx) {
                    const uint32_t room = m.stage_rows - nt;
                    if (ssrc[sidx] == HN_EMPTY || room == 0) continue;
                    bool c[2];
                    uint32_t r[2], snb[2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        c[h] = false; r[h] = 0;
                        const uint32_t slot = (uint32_t)lane + 32u * h;
                        const uint32_t nd = slot < take ? m.sadj[sidx * HN_MAX_TAKE + slot] : HN_EMPTY;
                        snb[h] = nd;
                        if (nd != HN_EMPTY) {
                            r[h] = node_row ? __ldg(node_row + nd) : nd;
                            const uint32_t id = hn_id(sc.root_row, r[h]);
                            const uint32_t b = (((id >> 6) & bmask) << 6) | (id & 0x3f);
                            if (((m.fs[b >> 5] >> (b & 31)) & 1u) == 0) c[h] = (uint32_t)(m.cache[hw_cache_slot(nd)] >> 32) != nd;
                        }
                    }
                    const uint32_t c0 = __ballot_sync(0xFFFFFFFFu, c[0]);
                    const uint32_t c1 = take > 32 ? __ballot_sync(0xFFFFFFFFu, c[1]) : 0u;
                    const uint32_t n0 = (uint32_t)__popc(c0), tot = n0 + (uint32_t)__popc(c1);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (c[h]) {
                            const uint32_t pch = (h ? n0 : 0u) + (uint32_t)__popc((h ? c1 : c0) & lt);
                            if (pch < room) {
                                m.wnode[nt + pch] = snb[h]; m.wrow[nt + pch] = r[h];
                                // a row scored ahead of time is accepted later WITHOUT a chain phase and may be the very next
                                // head: its adjacency slots must be on their way to L2 now, not when it is accepted
                                const uint8_t *ap = reinterpret_cast<const uint8_t *>(adj + (size_t)snb[h] * nb);
                                hw_prefetch_l2(ap);
                                if (nb > 32) hw_prefetch_l2(ap + 128);
                            }
                        }
                    if (tot <= room) { sd3 = sd2; sd2 = sd1; sd1 = sd0; sd0 = ssrc[sidx]; }   // nothing left to score for this entry
                    nt += min(tot, room);
                }
            }
            __syncwarp();   // work list visible
            if (PROF) { const long long tq = clock64(); st.prof[9] += tq - t3; st.prof[11] += nt - nm; t3 = tq; }
            if (nt) e = hw_score_work<FAST, PROF>(sc, m, qmag, pp, nm, nt, lane, st);
        } else {
            e = hw_score_group<FAST, PROF>(sc, m, qmag, pp, 0, nc, lane, st);
        }
        st.evals += nc;
        if (e != 0xFFFFFFFFu) { st.err = e & 0xFFu; st.rlen = rlen; return; }
        if (PROF) t4 = clock64();
        if (f_pool) {
            uint64_t *P = m.qkeys;
            uint32_t *PN = m.qnodes;
            // ---- append the new entries, pick the next head, keep the pool bounded
            if ((uint32_t)lane < nc) { P[qlen + lane] = m.nkeys[lane]; PN[qlen + lane] = m.nnodes[lane]; }
            if ((uint32_t)lane + 32u < nc) { P[qlen + lane + 32] = m.nkeys[lane + 32]; PN[qlen + lane + 32] = m.nnodes[lane + 32]; }
            qlen += nc;
            ++visited;
            __syncwarp();
            const uint32_t R = ef - visited;   // pops still to come
            have_head = false;
            pre_node = HN_EMPTY;
            if (R > 0 && qlen > 0) {
                uint64_t best = 0ull;
                uint32_t bidx = 0;
                for (uint32_t i = lane; i < qlen; i += 32) { const uint64_t k = P[i]; if (k > best) { best = k; bidx = i; } }
                const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, (uint32_t)(best >> 32));
                const uint32_t lo = __reduce_max_sync(0xFFFFFFFFu, (uint32_t)(best >> 32) == hi ? (uint32_t)best : 0u);
                const uint64_t mx = ((uint64_t)hi << 32) | lo;
                const uint32_t who = __ballot_sync(0xFFFFFFFFu, best == mx);
                const uint32_t idx = __shfl_sync(0xFFFFFFFFu, bidx, __ffs(who) - 1);
                hkey = mx;
                hnode = PN[idx];
                have_head = true;
                if (f_preload) {   // its adjacency slots travel while the pool is tidied up
                    pre_node = hnode;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t slot = (uint32_t)lane + 32u * h;
                        pre_nbl[h] = slot < take ? __ldg(adj + (size_t)hnode * nb + slot) : HN_EMPTY;
                    }
                }
                __syncwarp();
                if (lane == 0 && idx != qlen - 1) { P[idx] = P[qlen - 1]; PN[idx] = PN[qlen - 1]; }   // remove: last entry fills the hole
                --qlen;
                __syncwarp();
                if (qlen + HN_MAX_TAKE > CAPQ) {
                    // the next pop's up to 64 new entries might not fit: drop entries that can never be popped.  T is raised
                    // to pivots that still have >= R better entries; anything <= T is droppable.
                    uint64_t T = 0ull;
                    uint32_t kept = qlen;
                    for (uint32_t it = 0; it < 12 && kept + HN_MAX_TAKE + 32 > CAPQ; ++it) {
                        const uint64_t pivot = P[(visited * 7u + it * 61u) % qlen];
                        if (pivot <= T) continue;
                        uint32_t c = 0;
                        for (uint32_t i = lane; i < qlen; i += 32) c += P[i] > pivot;
                        c = __reduce_add_sync(0xFFFFFFFFu, c);
                        if (c >= R) { T = pivot; kept = c; }
                    }
                    if (kept + HN_MAX_TAKE > CAPQ) {
                        // unlucky pivots: exact selection of the R best (rank by counting), slow but always sufficient (R <= EFP)
                        for (uint32_t i0 = 0; i0 < qlen; i0 += 32) {
                            const uint32_t i = i0 + lane;
                            const uint64_t k = i < qlen ? P[i] : 0ull;
                            uint32_t rank = 0;
                            for (uint32_t j = 0; j < qlen; ++j) rank += P[j] > k;
                            const uint32_t cand = (i < qlen && rank == R - 1) ? 1u : 0u;   // the R-th best key
                            const uint32_t b = __ballot_sync(0xFFFFFFFFu, cand);
                            if (b) { const uint64_t kk = __shfl_sync(0xFFFFFFFFu, k, __ffs(b) - 1); T = kk - 1; }
                        }
                        if (qlen < R) T = 0ull;
                    }
                    // in-place stream compaction (destinations never overtake the rows still to be read)
                    uint32_t dst = 0;
                    for (uint32_t i0 = 0; i0 < qlen; i0 += 32) {
                        const uint32_t i = i0 + lane;
                        const uint64_t k = i < qlen ? P[i] : 0ull;
                        const uint32_t nd = i < qlen ? PN[i] : 0u;
                        const bool keep = i < qlen && k > T;
                        const uint32_t b = __ballot_sync(0xFFFFFFFFu, keep);
                        __syncwarp();
                        if (keep) { const uint32_t d = dst + (uint32_t)__popc(b & lt); P[d] = k; PN[d] = nd; }
                        dst += (uint32_t)__popc(b);
                        __syncwarp();
                    }
                    qlen = dst;
                }
            }
        } else
        // ---- merge the old queue (minus the popped head) with the new entries, keep what can still be popped.
        // Final position of an entry = number of entries of the union that are better; no sort of the new entries needed.
        {
            const uint32_t oldn = qlen - 1;
            const uint32_t cap = min(ef - (visited + 1), EFP);
            uint64_t *D = m.qkeys + (cur ^ 1) * EFP;
            uint32_t *DN = m.qnodes + (cur ^ 1) * EFP;
            const uint64_t mynk0 = (uint32_t)lane < nc ? m.nkeys[lane] : 0ull;
            const uint64_t mynk1 = (uint32_t)lane + 32u < nc ? m.nkeys[lane + 32] : 0ull;
            // the next head is the better of the runner-up and the best new entry: start loading its adjacency slots now,
            // the loads complete while the merge below runs
            pre_node = HN_EMPTY;
            if (f_preload && cap > 0 && oldn + nc > 0) {
                uint64_t best = oldn ? Q[1] : 0ull;
                uint32_t next = oldn ? QN[1] : HN_EMPTY;
                if (nc) {
                    // max of the (unique) 64-bit keys: two 32-bit warp reductions (REDUX) instead of a shuffle tree
                    const uint64_t loc = mynk0 > mynk1 ? mynk0 : mynk1;
                    const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, (uint32_t)(loc >> 32));
                    const uint32_t lo = __reduce_max_sync(0xFFFFFFFFu, (uint32_t)(loc >> 32) == hi ? (uint32_t)loc : 0u);
                    const uint64_t mx = ((uint64_t)hi << 32) | lo;
                    if (mx > best) {
                        const uint32_t who0 = __ballot_sync(0xFFFFFFFFu, mynk0 == mx), who1 = __ballot_sync(0xFFFFFFFFu, mynk1 == mx);
                        next = m.nnodes[who0 ? (uint32_t)__ffs(who0) - 1u : 32u + (uint32_t)__ffs(who1) - 1u];
                        best = mx;
                    }
                }
                pre_node = next;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t slot = (uint32_t)lane + 32u * h;
                    pre_nbl[h] = slot < take ? __ldg(adj + (size_t)next * nb + slot) : HN_EMPTY;
                }
            }
            uint32_t r0 = 0, r1 = 0;       // new entries better than my new entries
            if (oldn <= 128) {
                // every lane keeps 4 old entries in registers; one pass over the few new keys (broadcast reads) yields, for the
                // old entries, how far they move down and, through ballots, how many old entries beat each new one
                uint64_t ok[4];
                uint32_t lo[4] = {0, 0, 0, 0};
#pragma unroll
                for (int t = 0; t < 4; ++t) ok[t] = (uint32_t)lane + 32u * t < oldn ? Q[1 + lane + 32 * t] : 0ull;   // 0 = no entry (never better)
                uint32_t c0 = 0, c1 = 0;   // old entries better than my new entries (lane j & 31 keeps the count of new entry j)
                for (uint32_t j = 0; j < nc; ++j) {
                    const uint64_t nk = m.nkeys[j];
                    uint32_t cnt = 0;
#pragma unroll
                    for (int t = 0; t < 4; ++t) {   // keys are unique and "no entry" is 0: ok[t] > nk  <=>  !(nk > ok[t])
                        const bool gt = nk > ok[t];
                        lo[t] += gt;
                        cnt += 32u - (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, gt));
                    }
                    r0 += nk > mynk0;
                    r1 += nk > mynk1;
                    if (lane == (int)(j & 31)) { if (j < 32) c0 = cnt; else c1 = cnt; }
                }
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const uint32_t i = (uint32_t)lane + 32u * t;
                    const uint32_t pos = i + lo[t];
                    if (i < oldn && pos < cap) { D[pos] = ok[t]; DN[pos] = QN[1 + i]; }
                }
                if ((uint32_t)lane < nc && r0 + c0 < cap) { D[r0 + c0] = mynk0; DN[r0 + c0] = m.nnodes[lane]; }
                if ((uint32_t)lane + 32u < nc && r1 + c1 < cap) { D[r1 + c1] = mynk1; DN[r1 + c1] = m.nnodes[lane + 32]; }
            } else {
                // long queues (ef_search > 128): counting for the old entries, binary search in the sorted old queue for the new
                for (uint32_t i = lane; i < oldn; i += 32) {
                    const uint64_t k = Q[1 + i];
                    uint32_t lo = 0;
                    for (uint32_t j = 0; j < nc; ++j) lo += m.nkeys[j] > k;
                    const uint32_t pos = i + lo;
                    if (pos < cap) { D[pos] = k; DN[pos] = QN[1 + i]; }
                }
                for (uint32_t j = 0; j < nc; ++j) { const uint64_t nk = m.nkeys[j]; r0 += nk > mynk0; r1 += nk > mynk1; }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint32_t p = (uint32_t)lane + 32u * h;
                    if (p < nc) {
                        const uint64_t k = h ? mynk1 : mynk0;
                        uint32_t lo = 0, hi = oldn;  // number of old entries better than k
                        while (lo < hi) { const uint32_t md = (lo + hi) >> 1; if (Q[1 + md] > k) lo = md + 1; else hi = md; }
                        const uint32_t pos = (h ? r1 : r0) + lo;
                        if (pos < cap) { D[pos] = k; DN[pos] = m.nnodes[p]; }
                    }
                }
            }
            qlen = min(oldn + nc, cap);
            cur ^= 1;
            ++visited;
        }
        __syncwarp();
        if (PROF) {
            const long long t5 = clock64();
            st.prof[0] += t2 - t1; st.prof[1] += t3 - t2; st.prof[5] += t5 - t4;
        }
    }
    long long t6 = 0;
    if (PROF) t6 = clock64();
    uint32_t P = 1;
    while (P < rlen) P <<= 1;
    hw_sort_desc(m.rkeys, m.rnodes, rlen, P, lane);
    st.rlen = rlen;
    if (PROF) { const long long t7 = clock64(); st.prof[6] += t7 - t6; st.prof[7] += t7 - t0; }
}

template <int FAST, bool PROF>
__global__ void __launch_bounds__(32) hnsw_search_warp_kernel(HnswArgs a, HwCarve cv) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x;
    const uint32_t qi = blockIdx.x;
    HwSmem m;
    m.qs = smem;
    m.q32 = reinterpret_cast<float *>(smem + cv.off_q32);
    m.qkeys = reinterpret_cast<uint64_t *>(smem + cv.off_qkeys);
    m.rkeys = reinterpret_cast<uint64_t *>(smem + cv.off_rkeys);
    m.nkeys = reinterpret_cast<uint64_t *>(smem + cv.off_nkeys);
    m.fs = reinterpret_cast<uint32_t *>(smem + cv.off_fs);
    m.bar = hw_smem_u32(smem + cv.off_bar);
    m.qnodes = reinterpret_cast<uint32_t *>(smem + cv.off_qnodes);
    m.rnodes = reinterpret_cast<uint32_t *>(smem + cv.off_rnodes);
    m.nnodes = reinterpret_cast<uint32_t *>(smem + cv.off_nnodes);
    m.nrow = reinterpret_cast<uint32_t *>(smem + cv.off_nrow);
    m.stage = smem + cv.off_stage;
    m.cache = reinterpret_cast<uint64_t *>(smem + cv.off_cache);
    m.wnode = reinterpret_cast<uint32_t *>(smem + cv.off_work);
    m.wrow = m.wnode + HW_WORK;
    m.wdst = m.wrow + HW_WORK;
    m.sadj = reinterpret_cast<uint32_t *>(smem + cv.off_sadj);
    m.EFP = cv.EFP; m.stage_pitch = cv.stage_pitch; m.stage_rows = cv.stage_rows;

    for (uint32_t i = lane; i < a.row_pitch / 4; i += 32)
        reinterpret_cast<uint32_t *>(m.qs)[i] = reinterpret_cast<const uint32_t *>(a.q + (size_t)qi * a.row_pitch)[i];
    __syncwarp();
    const float qmag = a.qmags[qi];
    const HnScoreCtx sc{a.rows, a.row_pitch, a.mags, a.dim, a.st, a.metric, a.g.root_row};
    if (lane == 0) hw_mbar_init(m.bar, 1);
    HwState st;
    st.err = 0; st.rlen = 0; st.evals = 0; st.pops = 0; st.bar_phase = 0;
#pragma unroll
    for (int i = 0; i < HW_PROF_SLOTS; ++i) st.prof[i] = 0;
    uint32_t entry = a.g.entry, out_total = 0;
    __syncwarp();

    // ann_search (vector_store.rs:256-402): fresh fixed set and ef budget per level, results of all levels
    // concatenated, child of the best result is the entry of the next level
    for (int level = (int)a.g.num_levels; level >= 0; --level) {
        const uint32_t nb = level == 0 ? a.g.nbrs0 : a.g.nbrs;
        const uint32_t take = min(min(a.shortlist, nb), HN_MAX_TAKE);
        const uint32_t *node_row = ((a.g.identity_mask >> level) & 1u) ? nullptr : a.g.node_row[level];
        hw_traverse_level<FAST, PROF>(node_row, a.g.adj[level], nb, take, sc, m, qmag, HN_QUERY_ID, a.ef, entry, st, lane, a.flags);
        if (st.err) break;
        const uint32_t keep = min(st.rlen, HW_FINAL_LEN);
        for (uint32_t i = lane; i < keep; i += 32) {
            const uint32_t slot = out_total + i;
            if (slot < a.out_cap) {
                const uint32_t nd = m.rnodes[i];
                a.out_rows[(size_t)qi * a.out_cap + slot] = node_row ? node_row[nd] : nd;
                a.out_scores[(size_t)qi * a.out_cap + slot] = __uint_as_float(key_to_bits(a.metric, (uint32_t)(m.rkeys[i] >> 32)));
            }
        }
        out_total += keep;
        if (level > 0) entry = a.g.child[level][m.rnodes[0]];
        __syncwarp();
    }
    if (lane == 0) {
        a.out_n[qi] = st.err ? 0u : min(out_total, a.out_cap);
        if (st.err) atomicOr(a.err32 + qi, st.err);
        if (a.counters) { atomicAdd(a.counters, st.evals); atomicAdd(a.counters + 1, st.pops); }
        if (PROF && a.prof) {
            st.prof[8] = (long long)st.pops;
            for (int i = 0; i < HW_PROF_SLOTS; ++i) atomicAdd(a.prof + i, (unsigned long long)st.prof[i]);
        }
    }
}

static int hw_fast_kind(int st, int metric) {   // 1: f16 chain, 2: bf16 chain, 0: generic pair_distance
    if (metric != CDB_METRIC_COSINE && metric != CDB_METRIC_DOT_PRODUCT) return 0;
    return st == CDB_ST_F16 ? 1 : (st == CDB_ST_BF16 ? 2 : 0);
}
size_t hnsw_warp_smem(uint32_t row_pitch, uint32_t dim, uint32_t ef, int st, int metric) {
    return hw_carve(row_pitch, dim, ef, hw_fast_kind(st, metric) != 0, true).total;
}

template <int FAST, bool PROF>
static cdb_status launch_warp(const HnswArgs &a, const HwCarve &cv, cudaStream_t s) {
    auto kern = hnsw_search_warp_kernel<FAST, PROF>;
    CDB_ALLOW_SMEM(kern, cv.total);
    kern<<<a.nq, 32, cv.total, s>>>(a, cv);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

cdb_status hnsw_search_warp_device(const HnswArgs &a, cudaStream_t s) {
    if (!a.nq) return CDB_OK;
    if (a.ef == 0 || a.ef > 4096) { set_error("hnsw: ef_search must be in 1..4096"); return CDB_INVALID_PARAMS; }
    const int fast = hw_fast_kind(a.st, a.metric);
    const bool spec = (a.flags & CDB_HNSW_F_SPEC) != 0 && (a.flags & CDB_HNSW_F_POOL) == 0;
    const HwCarve cv = hw_carve(a.row_pitch, a.dim, a.ef, fast != 0, spec);
    if (cv.total > 200 * 1024) { set_error("hnsw: ef_search / row size too large for shared memory"); return CDB_INVALID_PARAMS; }
    const bool prof = a.prof != nullptr;
    if (fast == 1) return prof ? launch_warp<1, true>(a, cv, s) : launch_warp<1, false>(a, cv, s);
    if (fast == 2) return prof ? launch_warp<2, true>(a, cv, s) : launch_warp<2, false>(a, cv, s);
    return prof ? launch_warp<0, true>(a, cv, s) : launch_warp<0, false>(a, cv, s);
}

}  // namespace cdb
