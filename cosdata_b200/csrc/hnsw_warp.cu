// hnsw_warp.cu -- batched HNSW search, ONE WARP PER QUERY (S1, CDB_MODE_HNSW; graphs with metadata: the md form at the end):
//   ann_search              src/vector_store.rs:256-402
//   traverse_find_nearest   src/vector_store.rs:1112-1204 (hw_traverse_level, hnsw_traverse.cuh: why one warp per query)
#include "hnsw_traverse.cuh"

namespace cdb {

constexpr uint32_t HW_FINAL_LEN = 100;          // vector_store.rs:1194

template <int FAST, bool PROF>
__global__ void __launch_bounds__(32) hnsw_search_warp_kernel(HnswArgs a, HwCarve cv) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x;
    const uint32_t qi = blockIdx.x;
    const HwSmem m = hw_smem(smem, cv);

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
        hw_traverse_level<FAST, PROF, false>(node_row, a.g.adj[level], nb, take, sc, m, qmag, HN_QUERY_ID, true, a.ef, entry, st, lane);
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

template <int FAST, bool PROF>
static cdb_status launch_warp(const HnswArgs &a, const HwCarve &cv, cudaStream_t s) {
    auto kern = hnsw_search_warp_kernel<FAST, PROF>;
    CDB_ALLOW_SMEM(kern, cv.total);
    kern<<<a.nq, 32, cv.total, s>>>(a, cv);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

cdb_status hnsw_search_check(uint32_t row_pitch, uint32_t ef, bool md, uint32_t M) {
    if (ef == 0 || ef > 4096) { set_error("hnsw: ef_search must be in 1..4096"); return CDB_INVALID_PARAMS; }
    if (hw_carve(row_pitch, ef, md, M).total > 200 * 1024) {
        set_error(md ? "hnsw: ef_search / metadata dims too large for shared memory" : "hnsw: ef_search / row size too large for shared memory");
        return CDB_INVALID_PARAMS;
    }
    return CDB_OK;
}

cdb_status hnsw_search_warp_device(const HnswArgs &a, cudaStream_t s) {
    if (!a.nq) return CDB_OK;
    if (const cdb_status rc = hnsw_search_check(a.row_pitch, a.ef, false, 0)) return rc;
    const int fast = hw_fast_kind(a.st, a.metric);
    const HwCarve cv = hw_carve(a.row_pitch, a.ef);
    const bool prof = a.prof != nullptr;
    if (fast == 1) return prof ? launch_warp<1, true>(a, cv, s) : launch_warp<1, false>(a, cv, s);
    if (fast == 2) return prof ? launch_warp<2, true>(a, cv, s) : launch_warp<2, false>(a, cv, s);
    return prof ? launch_warp<0, true>(a, cv, s) : launch_warp<0, false>(a, cv, s);
}

// ---- metadata form: HNSW search with metadata filters on a flat graph with replica nodes (SURVEY 8f-4)
//   search_internal root selection        src/indexes/hnsw/mod.rs:411-420 (pseudo root when the query has a filter)
//   ann_search, filter branch + fallback  src/vector_store.rs:273-313, 329-380
//   CosineSimilarity::calculate arms      src/distance/cosine.rs:34-102 (metadata.cuh)
// Per level, one traversal per filter row, all of them on the level's fixed set; their <= 100 results minus the strong
// mismatches (cosine -1.0, vector_store.rs:294-303) are merged into the level's best-100 list z.  A level that ends empty
// scores its entry against every filter and keeps the strongest (vector_store.rs:329-380).  out_rows is CDB_INVALID_ID for
// pseudo nodes, out_ids the replica ids (hnsw_dedup_kernel and the re-rank take them unchanged).
// (32, 7): shared memory keeps 7 queries per SM at D = 768.  Stating that minimum lets ptxas hold the kernel's per-level state
// in registers; without it ptxas spilled that state around the chains' division calls.
template <int FAST>
__global__ void __launch_bounds__(32, 7) hnsw_search_warp_md_kernel(HnswMdArgs a, HwCarve cv) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x;
    const uint32_t qi = blockIdx.x;
    const HwSmem m = hw_smem(smem, cv);
    uint64_t *zkeys = reinterpret_cast<uint64_t *>(smem + cv.off_zkeys);
    uint32_t *znodes = reinterpret_cast<uint32_t *>(smem + cv.off_znodes);
    int32_t *qbits = reinterpret_cast<int32_t *>(smem + cv.off_qbits);
    // the filter rows [f0, f1) and the result count are touched once per level: they live in shared memory (volatile: re-read
    // there) instead of registers that ptxas would spill around the chains' division calls
    volatile uint32_t *qv = reinterpret_cast<uint32_t *>(smem + cv.off_qvars);
    const HnswArgs &g = a.a;
    const uint32_t lt = (1u << lane) - 1u;

    for (uint32_t i = lane; i < g.row_pitch / 4; i += 32)
        reinterpret_cast<uint32_t *>(m.qs)[i] = reinterpret_cast<const uint32_t *>(g.q + (size_t)qi * g.row_pitch)[i];
    const float qmag = g.qmags[qi];
    const HnScoreCtx sc{g.rows, g.row_pitch, g.mags, g.dim, g.st, g.metric, g.g.root_row};
    const uint32_t pp = plane_pitch(g.dim);
    if (lane == 0) hw_mbar_init(m.bar, 1);
    HwState st;
    st.err = 0; st.rlen = 0; st.evals = 0; st.pops = 0; st.bar_phase = 0;
    const bool hasf = a.has_filter && a.has_filter[qi];
    {
        uint32_t f0 = 0, f1 = 0;
        if (hasf && !hnm_filter_rows(a, qi, &f0, &f1)) st.err = CDB_ERRFLAG_BAD_FILTER;
        if (lane == 0) { qv[0] = f0; qv[1] = f1; qv[2] = 0; }
    }
    uint32_t entry = hasf ? a.pseudo_entry : g.g.entry;
    __syncwarp();

    // Metadata::from(&QueryFilterDimensions) (types.rs:127-146): mbits = dims as i32, mag = sqrt(sequential sum of squares);
    // every lane folds the same values in the same order
    auto load_filter = [&](uint32_t f) {
        __syncwarp();
        for (uint32_t i = lane; i < a.M; i += 32) qbits[i] = (int32_t)a.filter_dims[(size_t)f * a.M + i];
        __syncwarp();
        float t = 0.0f;
        for (uint32_t i = 0; i < a.M; ++i) { const float x = (float)qbits[i]; t = __fadd_rn(t, __fmul_rn(x, x)); }
        return __fsqrt_rn(t);
    };
    const uint32_t minus1 = order_key(CDB_METRIC_COSINE, __float_as_uint(-1.0f));

    for (int level = (int)g.g.num_levels; level >= 0 && !st.err; --level) {
        const uint32_t nb = level == 0 ? g.g.nbrs0 : g.g.nbrs;
        const uint32_t take = min(min(g.shortlist, nb), HN_MAX_TAKE);
        const uint32_t *node_row = g.g.node_row[level];
        HnMdCtx md{a.node_id[level], a.node_md[level], a.md_bits, a.md_mags, a.M, nullptr, 0.0f, false, false, 0u};
        uint32_t zn = 0;
        if (hasf) {
            for (uint32_t f = qv[0]; f < qv[1]; ++f) {
                md.q_mag = load_filter(f); md.q_bits = qbits; md.keep_fs = f > qv[0];
                hw_traverse_level<FAST, false, true>(node_row, g.g.adj[level], nb, take, sc, m, qmag, HN_QUERY_ID, true, g.ef, entry, st,
                                                     lane, &md);
                if (st.err) break;
                const uint32_t keep = min(st.rlen, HW_FINAL_LEN);
                for (uint32_t i0 = 0; i0 < keep; i0 += 32) {   // append in rank order; z is sorted below
                    const uint32_t i = i0 + (uint32_t)lane;
                    const uint64_t key = i < keep ? m.rkeys[i] : 0ull;
                    const bool app = i < keep && !(g.metric == CDB_METRIC_COSINE && (uint32_t)(key >> 32) == minus1);
                    const uint32_t b = __ballot_sync(0xFFFFFFFFu, app);
                    if (app) { const uint32_t pos = zn + (uint32_t)__popc(b & lt); zkeys[pos] = key; znodes[pos] = m.rnodes[i]; }
                    zn += (uint32_t)__popc(b);
                }
                __syncwarp();
                uint32_t P = 1;
                while (P < zn) P <<= 1;
                hw_sort_desc(zkeys, znodes, zn, P, lane);
                zn = min(zn, HW_FINAL_LEN);
            }
        } else {
            hw_traverse_level<FAST, false, true>(node_row, g.g.adj[level], nb, take, sc, m, qmag, HN_QUERY_ID, true, g.ef, entry, st, lane,
                                                 &md);
            if (!st.err) {
                zn = min(st.rlen, HW_FINAL_LEN);
                for (uint32_t i = lane; i < zn; i += 32) { zkeys[i] = m.rkeys[i]; znodes[i] = m.rnodes[i]; }
            }
        }
        if (st.err) break;
        if (zn == 0) {
            // the level's entry node itself, scored against every filter (not counted as an evaluation), strongest match kept
            uint64_t best = 0ull;
            bool have = false;
            for (uint32_t f = qv[0]; f < (hasf ? qv[1] : qv[0] + 1); ++f) {
                if (hasf) { md.q_mag = load_filter(f); md.q_bits = qbits; }
                if (lane == 0) { m.nnodes[0] = entry; m.nrow[0] = node_row[entry]; }
                __syncwarp();
                const uint32_t e = hw_score_group<FAST, false, true>(sc, m, qmag, pp, 0, 1, lane, st, &md);
                if (e != 0xFFFFFFFFu) { st.err = e & 0xFFu; break; }
                const uint64_t key = m.nkeys[0];   // same id every time: the score decides, the first maximum is kept
                if (!have || key > best) { best = key; have = true; }
            }
            if (st.err) break;
            if (!have) { st.err = CDB_ERRFLAG_UNREACHABLE; break; }   // Some(empty filter list): max().unwrap() panics
            __syncwarp();
            if (lane == 0) { zkeys[0] = best; znodes[0] = entry; }
            zn = 1;
            __syncwarp();
        }
        const uint32_t out_total = qv[2];
        for (uint32_t i = lane; i < zn; i += 32) {
            const uint32_t slot = out_total + i, node = znodes[i];
            if (slot < g.out_cap) {
                const size_t o = (size_t)qi * g.out_cap + slot;
                a.out_ids[o] = md.node_id[node];
                g.out_rows[o] = hnm_is_pseudo(a, level, node) ? CDB_INVALID_ID : node_row[node];
                g.out_scores[o] = __uint_as_float(key_to_bits(g.metric, (uint32_t)(zkeys[i] >> 32)));
            }
        }
        __syncwarp();
        if (lane == 0) qv[2] = out_total + zn;
        if (level > 0) entry = g.g.child[level][znodes[0]];
        __syncwarp();
    }
    if (lane == 0) {
        g.out_n[qi] = st.err ? 0u : min(qv[2], g.out_cap);
        if (st.err) atomicOr(g.err32 + qi, st.err);
        if (g.counters) { atomicAdd(g.counters, st.evals); atomicAdd(g.counters + 1, st.pops); }
    }
}

template <int FAST>
static cdb_status launch_warp_md(const HnswMdArgs &a, const HwCarve &cv, cudaStream_t s) {
    auto kern = hnsw_search_warp_md_kernel<FAST>;
    CDB_ALLOW_SMEM(kern, cv.total);
    kern<<<a.a.nq, 32, cv.total, s>>>(a, cv);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

cdb_status hnsw_search_md_device(const HnswMdArgs &a, cudaStream_t s) {
    if (!a.a.nq) return CDB_OK;
    if (const cdb_status rc = hnsw_search_check(a.a.row_pitch, a.a.ef, true, a.M)) return rc;
    const HwCarve cv = hw_carve(a.a.row_pitch, a.a.ef, true, a.M);
    const int fast = hw_fast_kind(a.a.st, a.a.metric);
    if (fast == 1) return launch_warp_md<1>(a, cv, s);
    if (fast == 2) return launch_warp_md<2>(a, cv, s);
    return launch_warp_md<0>(a, cv, s);
}

}  // namespace cdb
