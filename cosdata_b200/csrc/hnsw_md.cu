// hnsw_md.cu -- HNSW search with metadata filters on a flat graph with replica nodes (SURVEY 8f-4):
//   search_internal root selection        src/indexes/hnsw/mod.rs:411-420 (pseudo root when the query has a filter)
//   ann_search, filter branch + fallback  src/vector_store.rs:273-313, 329-380
//   CosineSimilarity::calculate arms      src/distance/cosine.rs:34-102 (metadata.cuh)
//   remove_duplicates_and_filter          src/models/common.rs:381-412 (dedup by replica id, pseudo nodes dropped)
//   get_raw_emb_by_internal_id            src/models/collection.rs:368-384 (replica id -> base vector; here node_row)
// One CTA per query; the traversal itself is the shared hn_traverse_level with a metadata context.  Searches run
// the warp-per-query form of the same steps (hnsw_warp.cu); this kernel answers CDB_HNSW_F_CTA and shapes whose warp carve
// does not fit.
// Per level and filter the <= 100 results are merged into the level's candidate list z (<= 100 best of all filters,
// vector_store.rs:306-312), entries scoring exactly -1.0 dropped (:294-303); the fixed set is shared by the filters of a level.
#include "hnsw_traverse.cuh"

namespace cdb {

constexpr uint32_t HNM_FINAL = 100;   // vector_store.rs:311, 1194
constexpr uint32_t HNM_Z = 256;       // z (<= 100) + one traversal (<= 100), padded for the bitonic sort

__global__ void __launch_bounds__(HN_THREADS) hnsw_search_md_kernel(HnswMdArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    const HnSmem m = hn_carve(smem, a.a.row_pitch, a.a.ef);
    uint64_t *zkeys = reinterpret_cast<uint64_t *>(smem + round_up((uint32_t)hn_smem_bytes(a.a.row_pitch, a.a.ef), 16));
    uint32_t *znodes = reinterpret_cast<uint32_t *>(zkeys + HNM_Z);
    int32_t *qbits = reinterpret_cast<int32_t *>(znodes + HNM_Z);
    __shared__ HnShared sh;
    __shared__ uint32_t s_zn, s_entry;
    __shared__ float s_fmag;
    const uint32_t qi = blockIdx.x;
    const int tid = threadIdx.x;
    const bool hasf = a.has_filter && a.has_filter[qi];
    uint32_t f0 = 0, f1 = 0;
    if (hasf && !hnm_filter_rows(a, qi, &f0, &f1)) {   // (uniform over the CTA: no barrier is skipped by part of it)
        if (tid == 0) { a.a.out_n[qi] = 0; atomicOr(a.a.err32 + qi, (uint32_t)CDB_ERRFLAG_BAD_FILTER); }
        return;
    }
    for (uint32_t i = tid; i < a.a.row_pitch / 4; i += HN_THREADS)
        reinterpret_cast<uint32_t *>(m.qs)[i] = reinterpret_cast<const uint32_t *>(a.a.q + (size_t)qi * a.a.row_pitch)[i];
    const float qmag = a.a.qmags[qi];
    const HnScoreCtx sc{a.a.rows, a.a.row_pitch, a.a.mags, a.a.dim, a.a.st, a.a.metric, a.a.g.root_row};
    if (tid == 0) { sh.err = 0; s_entry = hasf ? a.pseudo_entry : a.a.g.entry; }
    uint32_t out_total = 0;
    unsigned long long evals = 0, pops = 0;
    __syncthreads();

    // Metadata::from(&QueryFilterDimensions) (types.rs:127-146): mbits = dims as i32, mag = sqrt(sequential sum of squares)
    auto load_filter = [&](uint32_t f) {
        __syncthreads();
        for (uint32_t i = tid; i < a.M; i += HN_THREADS) qbits[i] = (int32_t)a.filter_dims[(size_t)f * a.M + i];
        __syncthreads();
        if (tid == 0) {
            float t = 0.0f;
            for (uint32_t i = 0; i < a.M; ++i) { const float x = (float)qbits[i]; t = __fadd_rn(t, __fmul_rn(x, x)); }
            s_fmag = __fsqrt_rn(t);
        }
        __syncthreads();
    };

    for (int level = (int)a.a.g.num_levels; level >= 0; --level) {
        const uint32_t nb = level == 0 ? a.a.g.nbrs0 : a.a.g.nbrs;
        const uint32_t take = min(min(a.a.shortlist, nb), HN_MAX_TAKE);
        const uint32_t *node_row = a.a.g.node_row[level];
        HnMdCtx md{a.node_id[level], a.node_md[level], a.md_bits, a.md_mags, a.M, nullptr, 0.0f, false};
        if (tid == 0) s_zn = 0;
        __syncthreads();
        if (hasf) {
            for (uint32_t f = f0; f < f1; ++f) {
                load_filter(f);
                md.q_bits = qbits; md.q_mag = s_fmag; md.keep_fs = f > f0;
                if (tid == 0) sh.entry = s_entry;
                __syncthreads();
                hn_traverse_level(node_row, a.a.g.adj[level], nb, take, sc, m, sh, qmag, HN_QUERY_ID, a.a.ef, evals, pops, &md);
                if (sh.err) break;
                const uint32_t keep = min(sh.rlen, HNM_FINAL);
                __syncthreads();
                // append what is not a strong mismatch (cs == -1.0, vector_store.rs:294-303); order is irrelevant, z is sorted below
                const uint32_t minus1 = order_key(CDB_METRIC_COSINE, __float_as_uint(-1.0f));
                for (uint32_t i = tid; i < keep; i += HN_THREADS) {
                    const uint64_t key = m.rkeys[i];
                    if (a.a.metric == CDB_METRIC_COSINE && (uint32_t)(key >> 32) == minus1) continue;
                    const uint32_t pos = atomicAdd(&s_zn, 1u);   // s_zn = entries kept so far (<= 100) + appended (<= 100)
                    zkeys[pos] = key; znodes[pos] = m.rnodes[i];
                }
                __syncthreads();
                const uint32_t total = s_zn;
                hn_sort_desc(zkeys, znodes, total, HNM_Z);
                if (tid == 0) s_zn = min(total, HNM_FINAL);
                __syncthreads();
            }
        } else {
            if (tid == 0) sh.entry = s_entry;
            __syncthreads();
            hn_traverse_level(node_row, a.a.g.adj[level], nb, take, sc, m, sh, qmag, HN_QUERY_ID, a.a.ef, evals, pops, &md);
            if (!sh.err) {
                const uint32_t keep = min(sh.rlen, HNM_FINAL);
                for (uint32_t i = tid; i < keep; i += HN_THREADS) { zkeys[i] = m.rkeys[i]; znodes[i] = m.rnodes[i]; }
                if (tid == 0) s_zn = keep;
            }
            __syncthreads();
        }
        if (sh.err) break;
        if (s_zn == 0) {
            // vector_store.rs:329-380: the level's entry node itself, scored against every filter, strongest match kept
            uint32_t best_key = 0, best_id = 0;
            bool have = false;
            for (uint32_t f = f0; f < (hasf ? f1 : f0 + 1); ++f) {
                if (hasf) { load_filter(f); md.q_bits = qbits; md.q_mag = s_fmag; }
                if (tid == 0 && !sh.err) {
                    float d = 0.f;
                    const int rc = hn_score_node(node_row, s_entry, sc, m, qmag, plane_pitch(sc.dim), &md, &d, &best_id);
                    if (rc != CDB_OK) sh.err = md_err_flag(rc);
                    const uint32_t k32 = order_key(sc.metric, __float_as_uint(d));
                    if (!have || k32 > best_key) { best_key = k32; have = true; }
                }
                __syncthreads();
                if (sh.err) break;
            }
            if (tid == 0 && !sh.err) {
                if (!have) sh.err = CDB_ERRFLAG_UNREACHABLE;   // Some(empty filter list): dists.into_iter().max().unwrap() panics
                else { zkeys[0] = make_key64(best_key, best_id); znodes[0] = s_entry; s_zn = 1; }
            }
            __syncthreads();
            if (sh.err) break;
        }
        const uint32_t zn = s_zn;
        for (uint32_t i = tid; i < zn; i += HN_THREADS) {
            const uint32_t slot = out_total + i, node = znodes[i];
            if (slot < a.a.out_cap) {
                const size_t o = (size_t)qi * a.a.out_cap + slot;
                a.out_ids[o] = a.node_id[level][node];
                a.a.out_rows[o] = hnm_is_pseudo(a, level, node) ? CDB_INVALID_ID : node_row[node];
                a.a.out_scores[o] = __uint_as_float(key_to_bits(a.a.metric, (uint32_t)(zkeys[i] >> 32)));
            }
        }
        out_total += zn;
        if (tid == 0 && level > 0) s_entry = a.a.g.child[level][znodes[0]];
        __syncthreads();
    }
    if (tid == 0) {
        a.a.out_n[qi] = sh.err ? 0u : min(out_total, a.a.out_cap);
        if (sh.err) atomicOr(a.a.err32 + qi, sh.err);
        if (a.a.counters) { atomicAdd(a.a.counters, evals); atomicAdd(a.a.counters + 1, pops); }
    }
}

// remove_duplicates_and_filter for replica nodes: first occurrence per replica id, root (id u32::MAX) and pseudo nodes
// (row == CDB_INVALID_ID) dropped, sorted best first, 5*k kept.  cand = id_base + vector row, labels = replica ids.
__global__ void __launch_bounds__(256) hnsw_dedup_md_kernel(const uint32_t *__restrict__ ids, const uint32_t *__restrict__ rows,
                                                            const float *__restrict__ scores, const uint32_t *__restrict__ n_in,
                                                            uint32_t in_cap, int metric, uint32_t id_base, uint32_t k5,
                                                            uint32_t *__restrict__ cand, uint32_t *__restrict__ labels,
                                                            uint32_t *__restrict__ cand_cnt) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *keys = reinterpret_cast<uint64_t *>(smem);
    uint32_t P = 1;
    while (P < in_cap) P <<= 1;
    uint32_t *vals = reinterpret_cast<uint32_t *>(keys + P);   // source position of the entry
    uint32_t *sid = vals + P;
    __shared__ int kept;
    const uint32_t q = blockIdx.x, n = min(n_in[q], in_cap);
    if (threadIdx.x == 0) kept = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) sid[i] = ids[(size_t)q * in_cap + i];
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t id = sid[i];
        bool dup = false;
        for (uint32_t j = 0; j < i; ++j) dup |= sid[j] == id;
        uint64_t key = 0;
        if (!dup && id != 0xFFFFFFFFu && rows[(size_t)q * in_cap + i] != CDB_INVALID_ID) {
            key = make_key64(order_key(metric, __float_as_uint(scores[(size_t)q * in_cap + i])), id);
            atomicAdd(&kept, 1);
        }
        keys[i] = key;
        vals[i] = i;
    }
    __syncthreads();
    for (uint32_t i = n + threadIdx.x; i < P; i += blockDim.x) { keys[i] = 0ull; vals[i] = 0; }
    __syncthreads();
    for (uint32_t size = 2; size <= P; size <<= 1)
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t x = keys[lo], y = keys[hi];
                if ((x < y) == desc) { keys[lo] = y; keys[hi] = x; const uint32_t v = vals[lo]; vals[lo] = vals[hi]; vals[hi] = v; }
            }
            __syncthreads();
        }
    const uint32_t mk = min((uint32_t)kept, k5);
    for (uint32_t i = threadIdx.x; i < mk; i += blockDim.x) {
        cand[(size_t)q * k5 + i] = id_base + rows[(size_t)q * in_cap + vals[i]];
        labels[(size_t)q * k5 + i] = sid[vals[i]];
    }
    if (threadIdx.x == 0) cand_cnt[q] = mk;
}

cdb_status hnsw_search_md_device(const HnswMdArgs &a, cudaStream_t s) {
    if (!a.a.nq) return CDB_OK;
    if (a.a.ef == 0 || a.a.ef > 4096) { set_error("hnsw: ef_search must be in 1..4096"); return CDB_INVALID_PARAMS; }
    const size_t smem = round_up((uint32_t)hn_smem_bytes(a.a.row_pitch, a.a.ef), 16) + (size_t)HNM_Z * 12 + (size_t)a.M * 4 + 16;
    if (smem > 200 * 1024) { set_error("hnsw: ef_search / metadata dims too large for shared memory"); return CDB_INVALID_PARAMS; }
    // the shapes accepted are this kernel's; the warp form takes every one of them whose own carve fits
    if (!(a.a.flags & CDB_HNSW_F_CTA) && hnsw_warp_md_smem(a.a.row_pitch, a.a.ef, a.M) <= 200 * 1024)
        return hnsw_search_warp_md_device(a, s);
    CDB_ALLOW_SMEM(hnsw_search_md_kernel, smem);
    hnsw_search_md_kernel<<<a.a.nq, HN_THREADS, smem, s>>>(a);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

cdb_status hnsw_dedup_md_device(const uint32_t *d_ids, const uint32_t *d_rows, const float *d_scores, const uint32_t *d_n,
                                uint32_t in_cap, int metric, uint32_t id_base, uint32_t k5, uint32_t nq, uint32_t *d_cand,
                                uint32_t *d_labels, uint32_t *d_cand_cnt, cudaStream_t s) {
    if (!nq) return CDB_OK;
    uint32_t P = 1;
    while (P < in_cap) P <<= 1;
    const size_t smem = (size_t)P * 12 + (size_t)in_cap * 4 + 16;
    if (smem > 200 * 1024) { set_error("hnsw dedup: too many levels"); return CDB_INVALID_PARAMS; }
    CDB_ALLOW_SMEM(hnsw_dedup_md_kernel, smem);
    hnsw_dedup_md_kernel<<<nq, 256, smem, s>>>(d_ids, d_rows, d_scores, d_n, in_cap, metric, id_base, k5, d_cand, d_labels, d_cand_cnt);
    CDB_LAUNCH_CHECK();
    return CDB_OK;
}

}  // namespace cdb
