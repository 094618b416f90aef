// hnsw_traverse.cuh -- traverse_find_nearest (src/vector_store.rs:1112-1204) on ONE WARP PER QUERY, shared by the searches
// (hnsw_warp.cu, plain graphs and graphs with metadata) and the graph writers' phase A (hnsw_build.cu: build, insert, delete).
//   PerformantFixedSet      src/models/fixedset.rs:2-29
//
// Keys are (order_key(score) << 32 | ~id) compared as u64: better score first, then smaller id (the oracle's tie rule where
// the reference's (MetricResult, pointer) order is unspecified).
//
// Why a warp.  A traversal is a chain of dependent pops; per pop only ~6 neighbours survive the fixed set, and each of
// them is scored by ONE thread because the reference arithmetic is a sequential chain per pair (dot_product_f16 is a
// left fold: 768 dependent adds).  The round-1 kernel gave every query a 128-thread CTA: three of its four warps waited
// at 9 block barriers per pop while one warp ran the chains (ncu: 63 % of warp samples parked at the barrier, 0.27 IPC on
// the scoring warp).  Here the 32 lanes of one warp ARE the neighbour slots (two slots per lane cover the <= 64 slots a
// pop examines), every hand-over is a __syncwarp / ballot / match, and the SM's four schedulers each see ~2 independent
// queries whose chains interleave.  Candidates, results, fixed set and the staged neighbour rows live in the warp's slice of
// shared memory (~24 KB at ef = 128, f16 x 768), so 7-9 queries are resident per SM -- all 1024 queries of a batch at once.
//
// Parity.  Pop order, fixed-set walk (slot order, aliasing ids included), first-Err rule, the (score, id) key and the
// per-level bookkeeping are the reference's; tests/test_gpu_hnsw.py checks ids, scores, counts, error flags AND the
// evaluation / pop counts against the oracle, and the writers' tests compare the graphs they build array for array.
//
// f16 chain.  dot_product_f16 = sum_i f32(x_i) * f32(y_i), sequential, no FMA in the reference.  The product of two
// halfs is exact in f32 (11 + 11 significand bits, exponent range far inside f32), so fma(x, y, s) rounds exactly once
// at the same place as s + (x * y): one fused multiply-add per element instead of FMUL + FADD, bit-identical.  The 16-bit
// operands are widened exactly from the packed registers (scorers.cuh, widen16), so no f32 query copy is needed.
#pragma once
#include "kernels.h"
#include "metadata.cuh"

namespace cdb {

constexpr uint32_t HN_EMPTY = 0xFFFFFFFFu;
constexpr uint32_t HN_ROOT_ID = 0xFFFFFFFFu;
constexpr uint32_t HN_QUERY_ID = 0xFFFFFFFEu;  // hnsw/mod.rs:398
constexpr uint32_t HN_MAX_TAKE = 64;            // slots examined per pop (<= shortlist_size, config.toml:32)

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
// staged neighbour rows per group, sized so that 7 warps (queries) per SM still fit in shared memory at D = 768:
constexpr uint32_t HW_STAGE_BYTES = 18700;      // 12 rows of f16 x 768, 6 of f32 x 768
// clock64 sums per query (lane 0): [0] pop + adjacency (+ node_row) loads, [1] fixed-set walk + compaction + prefetches,
// [2] issue of the row copies, [3] wait for the rows, [4] distance chains, [5] pool update (append, head, trim),
// [6] end-of-level result sort, [7] whole levels, [8] pops; counts: [9] pool trims, [10] of them by exact selection
constexpr int HW_PROF_SLOTS = 11;

constexpr uint32_t HW_MD_Z = 256;   // metadata form: a level's merged list z (<= 100) + one traversal's results (<= 100)

struct HwCarve {
    uint32_t EFP, stage_pitch, stage_rows;
    uint32_t off_qkeys, off_rkeys, off_nkeys, off_fs, off_qnodes, off_rnodes, off_nnodes, off_nrow, off_bar, off_stage, total;
    uint32_t off_zkeys, off_znodes, off_qvars, off_qbits; // metadata form only: z list, {f0, f1, results so far}, the filter's dims as i32 [M]
};

// md: metadata form with M metadata dims
__host__ __device__ inline HwCarve hw_carve(uint32_t row_pitch, uint32_t ef, bool md = false, uint32_t M = 0) {
    HwCarve c;
    c.EFP = hn_efp(ef);
    c.stage_pitch = round_up(row_pitch, 16) + 16;   // + 16 bytes: the lanes' rows start on different banks
    uint32_t r = HW_STAGE_BYTES / c.stage_pitch;
    c.stage_rows = r > 32 ? 32 : (r ? r : 1u);      // one lane scores one staged row
    uint32_t o = round_up(row_pitch, 16);           // the query's code (the chains widen it directly: no f32 copy)
    c.off_qkeys = o;          o += 2 * c.EFP * 8;
    c.off_rkeys = o;          o += c.EFP * 8;
    c.off_nkeys = o;          o += HN_MAX_TAKE * 8;
    c.off_bar = o;            o += 8;
    c.off_fs = o;             o += 128 * 4;
    c.off_qnodes = o;         o += 2 * c.EFP * 4;
    c.off_rnodes = o;         o += c.EFP * 4;
    c.off_nnodes = o;         o += HN_MAX_TAKE * 4;
    c.off_nrow = o;           o += HN_MAX_TAKE * 4;
    c.off_zkeys = c.off_znodes = c.off_qvars = c.off_qbits = 0;
    if (md) {
        o = round_up(o, 8);
        c.off_zkeys = o;      o += HW_MD_Z * 8;
        c.off_znodes = o;     o += HW_MD_Z * 4;
        c.off_qvars = o;      o += 4 * 4;
        c.off_qbits = o;      o += M * 4;
    }
    c.off_stage = round_up(o, 16);
    c.total = c.off_stage + c.stage_rows * c.stage_pitch;
    return c;
}

struct HwSmem {
    uint8_t *qs;
    uint64_t *qkeys, *rkeys, *nkeys;
    uint32_t *fs;            // PerformantFixedSet as 128 x 32-bit words: bucket b = words 2b, 2b+1 (native 32-bit shared atomics)
    uint32_t *qnodes, *rnodes, *nnodes, *nrow;
    uint8_t *stage;
    uint32_t bar;            // shared-space address of the warp's mbarrier (row copies complete on it)
    uint32_t EFP, stage_pitch, stage_rows;
};

__device__ __forceinline__ uint32_t hw_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
// TMA bulk copy (UBLKCP): `bytes` contiguous bytes global -> shared, completion counted on the mbarrier.  One instruction
// per row, issued by one lane: no per-lane address arithmetic, no LSU slots (16-byte cp.async would take 96 per f16 x 768 row).
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
__device__ __forceinline__ uint32_t hn_id(uint32_t root_row, uint32_t row) { return row == root_row ? HN_ROOT_ID : row; }

// metadata search: a pseudo node's results carry no vector row
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

__device__ __forceinline__ void hw_prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

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
// MD (metadata form): keys carry replica ids, and the metadata arm of each pair (md_arm) is applied first; a lane whose arm
// is a constant skips the chain.
template <int FAST, bool PROF, bool MD>
__device__ __forceinline__ uint32_t hw_score_group(const HnScoreCtx &sc, const HwSmem &m, float qmag, uint32_t pp, uint32_t first,
                                                   uint32_t n, int lane, HwState &st, const HnMdCtx *md) {
    uint32_t err_first = 0xFFFFFFFFu;
    for (uint32_t g0 = 0; g0 < n; g0 += m.stage_rows) {
        const uint32_t gn = min(m.stage_rows, n - g0);
        long long ts = 0, ti = 0, tw = 0;
        if (PROF) ts = clock64();
        uint32_t row = 0, nid = 0, mrow = HN_EMPTY;
        float rmag = 0.0f, ymag = 0.0f;
        // (a copy may complete before the expect_tx is posted: the phase cannot end before lane 0's arrive)
        if (lane == 0) hw_mbar_expect(m.bar, gn * sc.row_pitch);
        if ((uint32_t)lane < gn) {
            row = m.nrow[first + g0 + lane];
            hw_bulk_g2s(hw_smem_u32(m.stage + (size_t)lane * m.stage_pitch), sc.rows + (size_t)row * sc.row_pitch, sc.row_pitch, m.bar);
            rmag = sc.mags[row];   // in flight together with the rows
            if (MD) {
                const uint32_t node = m.nnodes[first + g0 + lane];
                nid = md->node_id[node];
                mrow = md->node_md[node];
                if (mrow != HN_EMPTY) ymag = md->md_mags[mrow];
            }
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
            int arm = MD_ARM_VECTOR;
            if (MD) {
                const MdSide x{m.qs, qmag, pp, md->q_has_id, md->q_id, md->q_bits, md->q_mag};
                const MdSide y{code, rmag, pp, true, nid, mrow == HN_EMPTY ? nullptr : md->md_bits + (size_t)mrow * md->M, ymag};
                arm = md_arm(sc.metric, md->M, x, y, &d);
                if (arm != MD_ARM_VECTOR) rc = arm;
            }
            if (arm == MD_ARM_VECTOR && FAST) {
                const float dot = hw_dot16<FAST>(m.qs, code, sc.dim);
                if (sc.metric == CDB_METRIC_COSINE) {
                    const float denom = __fmul_rn(qmag, rmag);
                    if (denom == 0.0f) rc = CDB_CALCULATION_ERROR;   // cosine.rs:230-231
                    else d = canon_nan(__fdiv_rn(dot, denom));
                } else {
                    d = dot;
                }
            } else if (arm == MD_ARM_VECTOR) {
                rc = pair_distance(sc.metric, sc.st, sc.dim, m.qs, qmag, pp, code, rmag, pp, &d);
            }
            m.nkeys[pos] = make_key64(order_key(sc.metric, __float_as_uint(d)), MD ? nid : hn_id(sc.root_row, row));
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

// One level (traverse_find_nearest).  All 32 lanes call it with warp-uniform arguments.  On return (st.err == 0)
// rkeys/rnodes[0..st.rlen) hold every popped entry sorted best first.  With seed_self, `self_id` is pre-inserted into the
// fixed set (the query id while searching, the new node's id while indexing: vector_store.rs:271, 807); a delete
// pre-inserts nothing (vector_store.rs:1231-1235).
// MD (metadata form, md != null): the fixed set and the keys use the replica ids md->node_id, pairs are scored through the
// metadata arms, md->keep_fs keeps the fixed set of the previous traversal of the level.
template <int FAST, bool PROF, bool MD>
__device__ void hw_traverse_level(const uint32_t *__restrict__ node_row /* null: identity */, const uint32_t *__restrict__ adj,
                                  uint32_t nb, uint32_t take, const HnScoreCtx &sc, const HwSmem &m, float qmag, uint32_t self_id,
                                  bool seed_self, uint32_t ef, uint32_t entry, HwState &st, int lane, const HnMdCtx *md = nullptr) {
    const uint32_t pp = plane_pitch(sc.dim);
    const uint32_t CAPQ = 2 * m.EFP;    // entries the candidate pool qkeys / qnodes holds
    const uint32_t bmask = nb - 1u;
    const uint32_t lt = (1u << lane) - 1u;
    long long t0 = 0;
    if (PROF) t0 = clock64();
    if (!MD || !md->keep_fs)
#pragma unroll
        for (int i = 0; i < 4; ++i) m.fs[lane + 32 * i] = 0u;
    if (lane == 0) { m.nnodes[0] = entry; m.nrow[0] = node_row ? node_row[entry] : entry; }
    __syncwarp();
    {
        const uint32_t e = hw_score_group<FAST, PROF, MD>(sc, m, qmag, pp, 0, 1, lane, st, md);
        st.evals += 1;
        if (e != 0xFFFFFFFFu) { st.err = e & 0xFFu; return; }
        if (lane == 0) {
            const uint32_t eid = MD ? md->node_id[entry] : hn_id(sc.root_row, m.nrow[0]);
            const uint32_t b0 = (((self_id >> 6) & bmask) << 6) | (self_id & 0x3f), b1 = (((eid >> 6) & bmask) << 6) | (eid & 0x3f);
            if (seed_self) m.fs[b0 >> 5] |= 1u << (b0 & 31);
            m.fs[b1 >> 5] |= 1u << (b1 & 31);
        }
        __syncwarp();
    }
    // The candidates other than the head are an UNSORTED pool in shared memory (qkeys / qnodes [0..qlen)), and each pop finds
    // the next head by an arg-max (8 slots per lane, two 32-bit REDUX).  The pop order is the reference heap's: the head is
    // the best entry present, and an entry is only ever dropped when at least (pops still to come) better entries exist, so
    // it could never have been popped.
    uint32_t qlen = 0, visited = 0, rlen = 0;
    uint64_t hkey = m.nkeys[0];
    uint32_t hnode = entry;
    bool have_head = true;
    // adjacency slots of the head, loaded one pop ahead (while the previous pop tidies up the pool)
    uint32_t pre_node = HN_EMPTY, pre_nbl[2] = {HN_EMPTY, HN_EMPTY};
    while (have_head) {   // false once the ef pops are done (R = 0 below) or the pool is empty
        long long t1 = 0, t2 = 0, t3 = 0, t4 = 0;
        if (PROF) t1 = clock64();
        // ---- pop
        const uint32_t bn = hnode;
        if (lane == 0) { m.rkeys[rlen] = hkey; m.rnodes[rlen] = bn; }
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
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            row[h] = 0;
            bk[h] = 0x80000000u | ((uint32_t)lane + 32u * h);   // unique per slot: never matches another slot
            if (nbl[h] != HN_EMPTY) {
                row[h] = node_row ? __ldg(node_row + nbl[h]) : nbl[h];
                const uint32_t id = MD ? __ldg(md->node_id + nbl[h]) : hn_id(sc.root_row, row[h]);
                bk[h] = (((id >> 6) & bmask) << 6) | (id & 0x3f);
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
            bool won0 = false, won1 = false;
            if (clear[0]) { const uint32_t bit = 1u << (bk[0] & 31); won0 = (atomicOr(&m.fs[bk[0] >> 5], bit) & bit) == 0; }
            if (clear[1]) { const uint32_t bit = 1u << (bk[1] & 31); won1 = (atomicOr(&m.fs[bk[1] >> 5], bit) & bit) == 0; }
            const uint32_t w0 = __ballot_sync(0xFFFFFFFFu, won0);
            const uint32_t w1 = two ? __ballot_sync(0xFFFFFFFFu, won1) : 0u;
            const bool resolve = __popc(w0) + __popc(w1) != __popc(cand0) + __popc(cand1);   // apply the slot-order rule explicitly
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
        const uint32_t e = hw_score_group<FAST, PROF, MD>(sc, m, qmag, pp, 0, nc, lane, st, md);
        st.evals += nc;
        if (e != 0xFFFFFFFFu) { st.err = e & 0xFFu; st.rlen = rlen; return; }
        if (PROF) t4 = clock64();
        // ---- append the new entries, pick the next head, keep the pool bounded
        uint64_t *P = m.qkeys;
        uint32_t *PN = m.qnodes;
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
            pre_node = hnode;   // its adjacency slots travel while the pool is tidied up
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t slot = (uint32_t)lane + 32u * h;
                pre_nbl[h] = slot < take ? __ldg(adj + (size_t)hnode * nb + slot) : HN_EMPTY;
            }
            __syncwarp();
            if (lane == 0 && idx != qlen - 1) { P[idx] = P[qlen - 1]; PN[idx] = PN[qlen - 1]; }   // remove: last entry fills the hole
            --qlen;
            __syncwarp();
            if (qlen + HN_MAX_TAKE > CAPQ) {
                // the next pop's up to 64 new entries might not fit: drop entries that can never be popped.  T is raised
                // to pivots that still have >= R better entries; anything <= T is droppable.
                if (PROF) st.prof[9] += 1;
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
                    if (PROF) st.prof[10] += 1;
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

__device__ __forceinline__ HwSmem hw_smem(uint8_t *smem, const HwCarve &cv) {
    HwSmem m;
    m.qs = smem;
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
    m.EFP = cv.EFP; m.stage_pitch = cv.stage_pitch; m.stage_rows = cv.stage_rows;
    return m;
}

inline int hw_fast_kind(int st, int metric) {   // 1: f16 chain, 2: bf16 chain, 0: generic pair_distance
    if (metric != CDB_METRIC_COSINE && metric != CDB_METRIC_DOT_PRODUCT) return 0;
    return st == CDB_ST_F16 ? 1 : (st == CDB_ST_BF16 ? 2 : 0);
}

}  // namespace cdb
