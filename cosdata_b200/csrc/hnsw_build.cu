// hnsw_build.cu -- GPU-side HNSW index build (SURVEY.md section 8f item 1): the write-side twin of hnsw.cu.
//   index_embeddings / index_embedding   src/vector_store.rs:714-940
//   create_node_edges                    src/vector_store.rs:976-1070
//   ProbNode::add_neighbor (+ eviction)  src/models/prob_node.rs:210-283
//   get_max_insert_level, level probs    src/models/common.rs:373-379, 421-429 (factor 4, api_service.rs:109)
// The reference builds concurrently (rayon batches racing through per-node locks), so its graph is not
// reproducible and parity is defined for SEARCH on a given graph (tests: the graph built here is exported and the
// CUDA search is compared with the oracle's search on it).  The build keeps the reference's algorithm:
//   phase A (hnsw_build_search_kernel): every vector of a batch runs traverse_find_nearest with ef_construction on
//     every level from the top (fixed set pre-seeded with its own id, best 64 kept) -- the same device code as the
//     search kernel -- against the graph as of the start of the batch;
//   phase B (hnsw_build_link_kernel): create_node_edges for levels 0..max_level with the reference's add_neighbor
//     (lowest-similarity slot, strict improvement, stale lowest_index, back-link removal of the evicted neighbour,
//     remove_neighbor_by_index_and_id on a failed reverse edge) under a per-node spin lock.
// A build is the root on every level followed by an insert of every row; cdb_index_insert_graph runs the same insert on
// rows appended later, against the slot state the build kept (or, for an uploaded graph, hnsw_slot_state_kernel derived).
// Batches grow geometrically from 1 so the upper structure is built almost sequentially.
// Level membership is decided up front (counter RNG or the caller's draws), so node_row / child are static during a call
// and only the adjacency (plus each slot's similarity and the node's lowest slot) evolves.
#include <algorithm>
#include <array>
#include <memory>
#include <unordered_map>
#include <vector>

#include "hnsw_traverse.cuh"

namespace cdb {

struct BuildLevel {
    uint32_t cnt, nb;
    uint32_t app;          // first node appended by the current call: level >= 1 lists its new rows ascending from here
    uint32_t *node_row;    // [cnt] (level >= 1: the root, then each call's rows ascending)
    uint32_t *child;       // [cnt] level-local index one level down
    uint32_t *adj;         // [cnt*nb]
    uint32_t *simkey;      // [cnt*nb] order key of the slot's similarity
    uint32_t *lowest_idx;  // [cnt]
    uint32_t *lowest_key;  // [cnt]
    int *lock;             // [cnt]
    // replica builds (collections with a metadata schema): [0] main root, [1] pseudo root, then created nodes in list order;
    // a graph attached by cdb_index_set_graph_slot_scores keeps its uploaded order, and the nodes each call appends follow
    const uint32_t *node_id;   // [cnt] ProbNode::get_id()
    const uint32_t *node_md;   // [cnt] metadata table row or HN_EMPTY
    const uint32_t *node_ins;  // [cnt] position in the replica list (roots HN_EMPTY); the current call's nodes ascend from `app`
};
constexpr int BUILD_MAX_LEVELS = 16;
struct BuildGraph {
    uint32_t num_levels, entry, root_row;
    BuildLevel lv[BUILD_MAX_LEVELS];
    uint32_t min_key, max_key;  // MetricResult::min / ::max as order keys (types.rs:435-457)
    uint32_t pseudo_entry;      // replica builds: top-level index of the pseudo root
};

// the flattened IndexableEmbeddings of preprocess_embedding (vector_store.rs:629-712) on the device
struct ReplicaDev {
    const uint32_t *row, *id, *base_id, *md;   // [n_nodes]
    const int32_t *md_bits;                    // [n_md][M]
    const float *md_mags;
    uint32_t M;
    uint32_t key_one, key_minus_one;           // order keys of cs == 1.0 / -1.0 (edge rules, vector_store.rs:1014-1040)
};

struct BuildArgs {
    BuildGraph g;
    HnScoreCtx sc;
    const uint8_t *levels;  // [count of the call] max insert level of row lv_first + i
    uint32_t lv_first;
    uint32_t first, count;  // rows [first, first+count) form this batch
    uint32_t ef, shortlist;
    uint32_t zcap;          // results kept per level: 64 (is_indexing) or 100 (delete_embedding)
    uint32_t *z_nodes;      // [count][num_levels+1][zcap]
    uint32_t *z_keys;       // [count][num_levels+1][zcap] order keys
    uint32_t *z_n;          // [count][num_levels+1] (delete: HN_EMPTY on the level whose traversal failed and below)
    uint8_t *failed;        // [count] 1: the traversal returned Err, 2: the row is deleted (not inserted)
    bool replicas;          // rows of the batch are positions of the replica list `rl`
    ReplicaDev rl;
    const uint32_t *deleted;   // deleted-row bitmap of the index (insert: such rows are skipped) or null
    const uint32_t *rowlist;   // delete: the batch is rows rowlist[first .. first+count), traversed on every level
};

__device__ __forceinline__ bool bit_set(const uint32_t *bits, uint32_t i) { return (bits[i >> 5] >> (i & 31)) & 1u; }

// local index of `row` at `level` (level 0: the row itself; level >= 1: binary search in the part of node_row the current
// call appended -- an uploaded level need not be sorted before it).  Replica graphs: `row` is a list position, searched among
// the nodes the current call created (they follow in list order from `app`)
__device__ inline uint32_t build_local(const BuildLevel &l, uint32_t level, uint32_t row, bool replicas = false) {
    if (replicas) {
        uint32_t lo = l.app, hi = l.cnt;
        while (lo < hi) { const uint32_t md = (lo + hi) >> 1; if (l.node_ins[md] < row) lo = md + 1; else hi = md; }
        return lo;
    }
    if (level == 0) return row;
    uint32_t lo = l.app, hi = l.cnt;
    while (lo < hi) { const uint32_t md = (lo + hi) >> 1; if (l.node_row[md] < row) lo = md + 1; else hi = md; }
    return lo;
}

// Phase A: one warp per entry of the batch runs the searches' traversal (hw_traverse_level) from the top level down.
// FAST = hw_fast_kind of the storage type and metric; MD = replica graph.  The traversal reads adj, node_row and node_id
// through the read-only cache (__ldg): node_row / node_id are fixed for the whole call, and the adjacency is written only by
// other launches on the same stream (phase B, the delete's repair and relink kernels), never while this kernel runs.
template <int FAST, bool MD>
__global__ void __launch_bounds__(32) hnsw_build_search_kernel(BuildArgs a, HwCarve cv) {
    extern __shared__ __align__(16) uint8_t smem[];
    const HwSmem m = hw_smem(smem, cv);
    const uint32_t b = blockIdx.x, r = a.rowlist ? a.rowlist[a.first + b] : a.first + b;
    const int lane = threadIdx.x;
    const bool del = a.rowlist != nullptr;
    if (!del && !MD && a.deleted && bit_set(a.deleted, r)) {   // a deleted row is not inserted
        if (lane == 0) a.failed[b] = 2;
        return;
    }
    const uint32_t vrow = MD ? a.rl.row[r] : r;
    for (uint32_t i = lane; i < a.sc.row_pitch / 4; i += 32)
        reinterpret_cast<uint32_t *>(m.qs)[i] = reinterpret_cast<const uint32_t *>(a.sc.rows + (size_t)vrow * a.sc.row_pitch)[i];
    const float qmag = a.sc.mags[vrow];
    const uint32_t max_level = del ? a.g.num_levels : a.levels[r - a.lv_first];
    const uint32_t L1 = a.g.num_levels + 1;
    // replica builds: the traversal carries the embedding's metadata and prop_value.id (vector_store.rs:809-821); nodes whose
    // metadata has mag != 0 (Pseudo / Metadata kinds) start at the pseudo root (:461-483, 755-758)
    HnMdCtx md{};
    uint32_t self_id = r;
    bool under_pseudo = false;
    if (MD) {
        const uint32_t mrow = a.rl.md[r];
        md.md_bits = a.rl.md_bits; md.md_mags = a.rl.md_mags; md.M = a.rl.M;
        md.q_bits = mrow == HN_EMPTY ? nullptr : a.rl.md_bits + (size_t)mrow * a.rl.M;
        md.q_mag = mrow == HN_EMPTY ? 0.0f : a.rl.md_mags[mrow];
        md.keep_fs = false; md.q_has_id = true; md.q_id = a.rl.base_id[r];
        self_id = a.rl.id[r];
        under_pseudo = md.q_bits && md.q_mag != 0.0f;
    }
    if (lane == 0) hw_mbar_init(m.bar, 1);
    HwState st;
    st.err = 0; st.rlen = 0; st.evals = 0; st.pops = 0; st.bar_phase = 0;
    uint32_t entry = under_pseudo ? a.g.pseudo_entry : a.g.entry;
    __syncwarp();
    for (int level = (int)a.g.num_levels; level >= 0; --level) {
        const BuildLevel &l = a.g.lv[level];
        const uint32_t take = min(min(a.shortlist, l.nb), HN_MAX_TAKE);
        if (MD) { md.node_id = l.node_id; md.node_md = l.node_md; }
        hw_traverse_level<FAST, false, MD>(l.node_row, l.adj, l.nb, take, a.sc, m, qmag, self_id, !del, a.ef, entry, st, lane,
                                           MD ? &md : nullptr);
        if (st.err) {
            if (del && lane == 0)   // D3: no relinks on this level or below
                for (int lv = level; lv >= 0; --lv) a.z_n[(size_t)b * L1 + lv] = HN_EMPTY;
            break;
        }
        const uint32_t keep = min(st.rlen, a.zcap);  // final_len: 64 while indexing, 100 otherwise (vector_store.rs:1194)
        if ((uint32_t)level <= max_level) {
            const size_t base = ((size_t)b * L1 + level) * a.zcap;
            for (uint32_t i = lane; i < keep; i += 32) {
                a.z_nodes[base + i] = m.rnodes[i];
                a.z_keys[base + i] = (uint32_t)(m.rkeys[i] >> 32);
            }
            if (lane == 0) a.z_n[(size_t)b * L1 + level] = keep;
        }
        if (level > 0) entry = l.child[m.rnodes[0]];
        __syncwarp();
    }
    if (lane == 0) a.failed[b] = st.err ? 1 : 0;  // the reference returns Err: the embedding is not indexed
}
using BuildSearchKernel = void (*)(BuildArgs, HwCarve);
constexpr BuildSearchKernel BUILD_SEARCH[3][2] = {   // [hw_fast_kind][replica graph]
    {hnsw_build_search_kernel<0, false>, hnsw_build_search_kernel<0, true>},
    {hnsw_build_search_kernel<1, false>, hnsw_build_search_kernel<1, true>},
    {hnsw_build_search_kernel<2, false>, hnsw_build_search_kernel<2, true>}};
static BuildSearchKernel build_search_kernel(const HnScoreCtx &sc, bool replicas) {
    return BUILD_SEARCH[hw_fast_kind(sc.st, sc.metric)][replicas ? 1 : 0];
}

__device__ inline void node_lock(int *lk) {
    while (atomicCAS(lk, 0, 1) != 0) __nanosleep(32);
    __threadfence();
}
__device__ inline void node_unlock(int *lk) {
    __threadfence();
    atomicExch(lk, 0);
}

// ProbNode::add_neighbor; returns the slot index or -1
__device__ int build_add_neighbor(const BuildGraph &g, const BuildLevel &l, uint32_t node, uint32_t nbr, uint32_t dkey) {
    volatile uint32_t *adj = l.adj + (size_t)node * l.nb;
    volatile uint32_t *sk = l.simkey + (size_t)node * l.nb;
    node_lock(l.lock + node);
    const uint32_t lidx = ((volatile uint32_t *)l.lowest_idx)[node], lkey = ((volatile uint32_t *)l.lowest_key)[node];
    if (dkey <= lkey) { node_unlock(l.lock + node); return -1; }
    bool ok = false;
    uint32_t old = HN_EMPTY;
    if (adj[lidx] == HN_EMPTY) { adj[lidx] = nbr; sk[lidx] = dkey; ok = true; }
    else if (dkey > sk[lidx]) { old = adj[lidx]; adj[lidx] = nbr; sk[lidx] = dkey; ok = true; }
    uint32_t nidx = 0, nkey = g.max_key;
    for (uint32_t s = 0; s < l.nb; ++s) {
        if (adj[s] == HN_EMPTY) { nkey = g.min_key; nidx = s; break; }
        const uint32_t k = sk[s];
        if (k < nkey) { nkey = k; nidx = s; }
    }
    ((volatile uint32_t *)l.lowest_idx)[node] = nidx;
    ((volatile uint32_t *)l.lowest_key)[node] = nkey;
    node_unlock(l.lock + node);
    if (!ok) return -1;
    if (old != HN_EMPTY) {  // the evicted neighbour drops its back link (remove_neighbor_by_id), lowest_index left stale
        volatile uint32_t *oa = l.adj + (size_t)old * l.nb;
        node_lock(l.lock + old);
        for (uint32_t s = 0; s < l.nb; ++s)
            if (oa[s] == node) { oa[s] = HN_EMPTY; break; }
        node_unlock(l.lock + old);
    }
    return (int)lidx;
}

// ProbNode::replica_node_kind (prob_node.rs:487-496): the node's own id and metadata
__device__ inline int build_node_kind(const ReplicaDev &rl, const BuildLevel &l, uint32_t node) {
    const uint32_t mrow = l.node_md[node];
    if (mrow == HN_EMPTY || rl.md_mags[mrow] == 0.0f) return MD_KIND_BASE;
    const uint32_t id = l.node_id[node];
    return id >= MD_PSEUDO_ID_LO && id <= MD_PSEUDO_ID_HI ? MD_KIND_PSEUDO : MD_KIND_METADATA;
}

// one warp per new vector, lane 0 works (a thread spinning on a lock must not share a warp with its holder)
__global__ void __launch_bounds__(128) hnsw_build_link_kernel(BuildArgs a) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if ((threadIdx.x & 31) != 0 || b >= a.count || a.failed[b]) return;
    const uint32_t r = a.first + b;
    const uint32_t L1 = a.g.num_levels + 1;
    const uint32_t top = min((uint32_t)a.levels[r - a.lv_first], a.g.num_levels);
    for (uint32_t level = 0; level <= top; ++level) {  // edges are created bottom-up as the recursion unwinds
        const BuildLevel &l = a.g.lv[level];
        const uint32_t node = build_local(l, level, r, a.replicas);
        const size_t base = ((size_t)b * L1 + level) * a.zcap;
        const uint32_t zn = a.z_n[(size_t)b * L1 + level];
        const bool rules = a.replicas && a.sc.metric == CDB_METRIC_COSINE;   // the rules match MetricResult::CosineSimilarity only
        const int nk = rules ? build_node_kind(a.rl, l, node) : MD_KIND_BASE;
        uint32_t successful = 0;
        for (uint32_t i = 0; i < zn; ++i) {
            if (successful >= l.nb) break;
            const uint32_t nbr = a.z_nodes[base + i], dkey = a.z_keys[base + i];
            if (rules && nk == MD_KIND_METADATA) {   // vector_store.rs:1014-1040
                const int bk = build_node_kind(a.rl, l, nbr);
                if (bk == MD_KIND_PSEUDO && dkey != a.rl.key_one) continue;          // pseudo neighbour: perfect match only
                if (bk == MD_KIND_METADATA && dkey == a.rl.key_minus_one) continue;  // metadata neighbour: not on a strong mismatch
            }
            const int idx = build_add_neighbor(a.g, l, node, nbr, dkey);
            if (idx >= 0) {
                const int j = build_add_neighbor(a.g, l, nbr, node, dkey);
                if (j >= 0) successful++;
                else {  // remove_neighbor_by_index_and_id
                    volatile uint32_t *na = l.adj + (size_t)node * l.nb;
                    node_lock(l.lock + node);
                    if (na[idx] == nbr) na[idx] = HN_EMPTY;
                    node_unlock(l.lock + node);
                }
            }
        }
    }
}

__global__ void fill_u32_kernel(uint32_t *p, uint32_t v, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ------------------------------------------------------------------ lowest_index of a loaded node
// ProbNode::new_with_neighbors_and_versions (prob_node.rs:155-169), over one node's slots held by a whole warp: each lane
// notes the slots it holds, finish() reduces.  The first empty slot gives MetricResult::min; otherwise, scanning from
// MetricResult::max, the first slot with a strictly lower key.
struct SlotLowest {
    uint32_t first_empty = HN_EMPTY;
    uint64_t best = ~0ull;   // (key << 32 | slot): lowest filled slot strictly below MetricResult::max
    __device__ void note(uint32_t s, bool empty, uint32_t key, uint32_t max_key) {
        if (empty) first_empty = min(first_empty, s);
        else if (key < max_key) best = min(best, ((uint64_t)key << 32) | s);
    }
    __device__ void finish(uint32_t min_key, uint32_t max_key, uint32_t &li, uint32_t &lk) {   // whole warp, every lane gets it
        for (int o = 16; o; o >>= 1) {
            best = min(best, (uint64_t)__shfl_xor_sync(0xFFFFFFFFu, best, o));
            first_empty = min(first_empty, __shfl_xor_sync(0xFFFFFFFFu, first_empty, o));
        }
        li = 0; lk = max_key;
        if (first_empty != HN_EMPTY) { li = first_empty; lk = min_key; }
        else if (best != ~0ull) { li = (uint32_t)best; lk = (uint32_t)(best >> 32); }
    }
};

// ------------------------------------------------------------------ slot state of an uploaded graph
// ProbNode::new_with_neighbors_and_versions (prob_node.rs:145-181): every slot's similarity is recomputed and lowest_index is
// the first empty slot (MetricResult::min) or else the first slot with a strictly lower similarity, scanning from
// MetricResult::max.  The builder stores the similarity of the NEW node (x) against the neighbour (y) on both ends of an
// edge; recomputing it from the node's side gives the same bits because every plain arm is symmetric.  A slot whose pair
// is an Err (a zero-norm row under cosine) cannot come from the reference's build: it gets MetricResult::min, so it is the
// first slot add_neighbor replaces.
// One warp per node: lane 0 stages the node's row, every lane with a filled slot stages that neighbour's row (TMA bulk
// copies completing on the warp's mbarrier, as hnsw_warp.cu stages rows), then lane s scores slot s with the same
// pair_distance every other scorer uses.  Slots go in rounds of `group` lanes when the rows of all 32 do not fit.
constexpr int SS_WARPS = 4;
constexpr uint32_t SS_STAGE_BYTES = 24 * 1024;   // shared memory per warp (node row + one round of neighbour rows)

__global__ void __launch_bounds__(SS_WARPS * 32) hnsw_slot_state_kernel(BuildLevel l, HnScoreCtx sc, uint32_t min_key, uint32_t max_key,
                                                                        uint32_t group) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t bars[SS_WARPS];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *own = smem + (size_t)warp * (group + 1) * sc.row_pitch;
    uint8_t *mine_row = own + (size_t)(lane + 1) * sc.row_pitch;
    const uint32_t bar = hw_smem_u32(&bars[warp]);
    if (lane == 0) hw_mbar_init(bar, 1);
    __syncwarp();
    const uint32_t pp = plane_pitch(sc.dim);
    uint32_t parity = 0;
    for (uint32_t node = blockIdx.x * SS_WARPS + warp; node < l.cnt; node += gridDim.x * SS_WARPS) {
        const uint32_t row = l.node_row[node];
        SlotLowest lo;
        for (uint32_t base = 0; base < l.nb; base += group) {
            const uint32_t s = base + lane;
            const bool in_round = lane < group && s < l.nb;
            const uint32_t nbr = in_round ? l.adj[(size_t)node * l.nb + s] : HN_EMPTY;
            const uint32_t filled = __ballot_sync(0xFFFFFFFFu, nbr != HN_EMPTY);
            if (in_round && nbr == HN_EMPTY) lo.note(s, true, 0, max_key);
            const uint32_t nrow = nbr != HN_EMPTY ? l.node_row[nbr] : 0;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the previous round's reads before the copies below
            __syncwarp();
            if (lane == 0) {
                hw_mbar_expect(bar, (uint32_t)(__popc(filled) + (base == 0)) * sc.row_pitch);
                if (base == 0) hw_bulk_g2s(hw_smem_u32(own), sc.rows + (size_t)row * sc.row_pitch, sc.row_pitch, bar);
            }
            __syncwarp();
            if (nbr != HN_EMPTY) hw_bulk_g2s(hw_smem_u32(mine_row), sc.rows + (size_t)nrow * sc.row_pitch, sc.row_pitch, bar);
            hw_mbar_wait(bar, parity);
            parity ^= 1u;
            if (nbr != HN_EMPTY) {
                float d = 0.f;
                const int rc = pair_distance(sc.metric, sc.st, sc.dim, own, sc.mags[row], pp, mine_row, sc.mags[nrow], pp, &d);
                const uint32_t key = rc == CDB_OK ? order_key(sc.metric, __float_as_uint(d)) : min_key;
                l.simkey[(size_t)node * l.nb + s] = key;
                lo.note(s, false, key, max_key);
            }
        }
        uint32_t li, lk;
        lo.finish(min_key, max_key, li, lk);
        if (lane == 0) {
            l.lowest_idx[node] = li;
            l.lowest_key[node] = lk;
        }
    }
}

// ------------------------------------------------------------------ host
struct HnswBuildState {
    BuildGraph g{};                          // level arrays (owned by the graph's allocations) and the slot state
    uint64_t cap[BUILD_MAX_LEVELS] = {};     // nodes each level's arrays hold
    // replica graphs (cdb_index_build_graph_replicas): levels also carry node_id / node_md / node_ins
    bool replicas = false;
    uint32_t n_list = 0;                     // replica list positions created so far (the next node's node_ins)
    uint32_t pseudo_root_row = 0;            // g.root_row is the main root's row
    uint32_t n_md = 0, md_dims = 0;          // the Metadata table (owned by the graph's allocations)
    const int32_t *md_bits = nullptr;
    const float *md_mags = nullptr;
};
void hnsw_state_free(HnswBuildState *st) { delete st; }
const uint32_t *hnsw_state_slot_keys(const HnswBuildState *st, uint32_t level) { return st->g.lv[level].simkey; }
bool hnsw_state_replica_info(const HnswBuildState *st, uint32_t *pseudo_root_row, uint32_t *n_md) {
    if (!st || !st->replicas) return false;
    *pseudo_root_row = st->pseudo_root_row;
    *n_md = st->n_md;
    return true;
}

static void metric_key_range(int metric, uint32_t *min_key, uint32_t *max_key) {   // MetricResult::min / ::max (types.rs:435-457)
    switch (metric) {
    case CDB_METRIC_COSINE: *min_key = order_key(metric, 0xBF800000u /* -1.0 */); *max_key = order_key(metric, 0x40000000u /* 2.0 */); break;
    default: *min_key = order_key(metric, 0xFF800000u /* -inf */); *max_key = order_key(metric, 0x7F800000u /* +inf */); break;
    }
}

static float unit_rng(uint64_t seed, uint64_t i) {  // stands in for rand::random::<f32>() (vector_store.rs:750-753)
    uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}
// get_max_insert_level with probabilities 1 - 4^-n: x >= 1 - 4^-lv is monotone in lv, so the largest satisfied lv is the
// first hit of the reference's top-down scan
static uint8_t draw_level(uint64_t seed, uint32_t row, uint32_t num_levels) {
    const double x = (double)unit_rng(seed, row);
    uint32_t ml = 0;
    double p4 = 1.0;
    for (uint32_t lv = 1; lv <= num_levels; ++lv) { p4 *= 4.0; if (x >= 1.0 - 1.0 / p4) ml = lv; else break; }
    return (uint8_t)ml;
}

static cdb_status publish(const HnswBuildState &st, const GraphHost &gh);

// device allocations freed when the owner goes out of scope (release() hands them over)
struct DevAllocs {
    std::vector<void *> p;
    ~DevAllocs() { for (void *q : p) cudaFree(q); }
    cdb_status get(void **out, size_t bytes) {
        CDB_CUDA_TRY(cudaMalloc(out, bytes ? bytes : 4));
        p.push_back(*out);
        return CDB_OK;
    }
    void release() { p.clear(); }
};

// the arrays of one level: per node (node_row, lowest_idx, lowest_key, lock, child), per slot (adj, simkey), and on replica
// graphs per node (node_id, node_md, node_ins)
constexpr int LEVEL_ARRAYS = 10, PLAIN_LEVEL_ARRAYS = 7;
static uint32_t *&level_array(BuildLevel &l, int t) {
    switch (t) {
    case 0: return l.node_row;
    case 1: return l.lowest_idx;
    case 2: return l.lowest_key;
    case 3: return reinterpret_cast<uint32_t *&>(l.lock);
    case 4: return l.child;
    case 5: return l.adj;
    case 6: return l.simkey;
    case 7: return const_cast<uint32_t *&>(l.node_id);
    case 8: return const_cast<uint32_t *&>(l.node_md);
    default: return const_cast<uint32_t *&>(l.node_ins);
    }
}
static size_t level_words(const BuildLevel &l, int t, uint64_t nodes) { return t == 5 || t == 6 ? nodes * l.nb : nodes; }

void hnsw_state_release(HnswBuildState *st, std::vector<void *> *allocs) {
    if (!st) return;
    auto drop = [&](const void *p) {
        auto it = p ? std::find(allocs->begin(), allocs->end(), p) : allocs->end();
        if (it == allocs->end()) return;
        allocs->erase(it);
        cudaFree(const_cast<void *>(p));
    };
    for (uint32_t L = 0; L <= st->g.num_levels && L < (uint32_t)BUILD_MAX_LEVELS; ++L)
        for (int t : {1, 2, 3, 6, 7, 8, 9}) drop(level_array(st->g.lv[L], t));   // not node_row / child / adj: the graph's
    drop(st->md_bits);
    drop(st->md_mags);
    delete st;
}

// the per-level columns of nodes appended to a replica graph, parallel to append_levels' rows
struct ReplicaCols {
    std::vector<std::vector<uint32_t>> id, md, ins;
};

// Appends nodes (vector rows rows[L], level-local children child[L] on levels >= 1; on replica graphs also rc->id / md / ins)
// to every level.  Arrays that must grow are allocated first (by half their size at least; level 0 never beyond rows_cap
// nodes): if one allocation fails, nothing has changed.  After that *changed is set; the old arrays are copied, the new
// nodes start as ProbNode::new (no neighbours, lowest_index (0, MetricResult::min)), the search layout is re-published and
// the old arrays are freed.
static cdb_status append_levels(HnswBuildState &st, const GraphHost &gh, const std::vector<std::vector<uint32_t>> &rows,
                                const std::vector<std::vector<uint32_t>> &child, uint64_t rows_cap, bool *changed, cudaStream_t s,
                                const ReplicaCols *rcols = nullptr) {
    const int n_arrays = st.replicas ? LEVEL_ARRAYS : PLAIN_LEVEL_ARRAYS;
    const uint32_t L1 = st.g.num_levels + 1;
    cdb_status rc;
    std::vector<uint64_t> cap(L1, 0);
    std::vector<std::array<uint32_t *, LEVEL_ARRAYS>> fresh(L1);
    DevAllocs grown;
    for (uint32_t L = 0; L < L1; ++L) {
        const BuildLevel &l = st.g.lv[L];
        fresh[L].fill(nullptr);
        const uint64_t need = (uint64_t)l.cnt + rows[L].size();
        if (need <= st.cap[L]) continue;
        cap[L] = std::max<uint64_t>(need, st.cap[L] + st.cap[L] / 2);
        if (L == 0) cap[L] = std::max<uint64_t>(need, std::min<uint64_t>(cap[L], rows_cap));
        for (int t = 0; t < n_arrays; ++t)
            if ((t != 4 || L > 0) && (rc = grown.get((void **)&fresh[L][t], level_words(l, t, cap[L]) * 4))) return rc;
    }
    // ---- commit: every new array joins the graph's allocations, the old ones leave them once the tables moved on
    *changed = true;
    gh.allocs->insert(gh.allocs->end(), grown.p.begin(), grown.p.end());
    grown.release();
    std::vector<void *> retired;
    for (uint32_t L = 0; L < L1; ++L) {
        BuildLevel &l = st.g.lv[L];
        if (cap[L]) {
            for (int t = 0; t < n_arrays; ++t) {
                if (!fresh[L][t]) continue;
                uint32_t *&arr = level_array(l, t);
                const size_t used = level_words(l, t, l.cnt);
                if (arr && used) CDB_CUDA_TRY(cudaMemcpyAsync(fresh[L][t], arr, used * 4, cudaMemcpyDeviceToDevice, s));
                if (arr) retired.push_back(arr);
                arr = fresh[L][t];
            }
            st.cap[L] = cap[L];
        }
        l.app = l.cnt;
        const uint32_t add = (uint32_t)rows[L].size();
        if (!add) continue;
        for (uint32_t i = 0; L > 0 && i < add; ++i)   // an uploaded level that listed node i as row i may stop doing so
            if (rows[L][i] != l.cnt + i) { gh.dev->identity_mask &= ~(1u << L); break; }
        CDB_CUDA_TRY(cudaMemcpyAsync(l.node_row + l.cnt, rows[L].data(), (size_t)add * 4, cudaMemcpyHostToDevice, s));
        if (L > 0) CDB_CUDA_TRY(cudaMemcpyAsync(l.child + l.cnt, child[L].data(), (size_t)add * 4, cudaMemcpyHostToDevice, s));
        if (rcols) {
            const std::vector<uint32_t> *col[3] = {&rcols->id[L], &rcols->md[L], &rcols->ins[L]};
            for (int c = 0; c < 3; ++c)
                CDB_CUDA_TRY(cudaMemcpyAsync(level_array(l, 7 + c) + l.cnt, col[c]->data(), (size_t)add * 4, cudaMemcpyHostToDevice, s));
        }
        const uint64_t slots = (uint64_t)add * l.nb;
        fill_u32_kernel<<<(uint32_t)((slots + 255) / 256), 256, 0, s>>>(l.adj + (size_t)l.cnt * l.nb, HN_EMPTY, slots);
        CDB_LAUNCH_CHECK();
        CDB_CUDA_TRY(cudaMemsetAsync(l.simkey + (size_t)l.cnt * l.nb, 0, slots * 4, s));
        CDB_CUDA_TRY(cudaMemsetAsync(l.lowest_idx + l.cnt, 0, (size_t)add * 4, s));
        fill_u32_kernel<<<(add + 255) / 256, 256, 0, s>>>(l.lowest_key + l.cnt, st.g.min_key, add);
        CDB_LAUNCH_CHECK();
        CDB_CUDA_TRY(cudaMemsetAsync(l.lock + l.cnt, 0, (size_t)add * 4, s));
        l.cnt += add;
    }
    CDB_CUDA_TRY(cudaStreamSynchronize(s));   // the copies are done (host vectors, old arrays)
    if ((rc = publish(st, gh))) return rc;
    for (void *p : retired) {
        gh.allocs->erase(std::find(gh.allocs->begin(), gh.allocs->end(), p));
        cudaFree(p);
    }
    return CDB_OK;
}

// points the search layout (pointer tables, counts, host copies) at the level arrays of `st`
static cdb_status publish(const HnswBuildState &st, const GraphHost &gh) {
    const uint32_t L1 = st.g.num_levels + 1;
    gh.cnt->assign(L1, 0);
    gh.nr->assign(L1, nullptr); gh.ad->assign(L1, nullptr); gh.ch->assign(L1, nullptr);
    for (uint32_t L = 0; L < L1; ++L) {
        (*gh.cnt)[L] = st.g.lv[L].cnt;
        (*gh.nr)[L] = st.g.lv[L].node_row;
        (*gh.ad)[L] = st.g.lv[L].adj;
        (*gh.ch)[L] = L ? st.g.lv[L].child : nullptr;
    }
    CDB_CUDA_TRY(cudaMemcpy((void *)gh.dev->node_row, gh.nr->data(), L1 * sizeof(void *), cudaMemcpyHostToDevice));
    CDB_CUDA_TRY(cudaMemcpy((void *)gh.dev->adj, gh.ad->data(), L1 * sizeof(void *), cudaMemcpyHostToDevice));
    CDB_CUDA_TRY(cudaMemcpy((void *)gh.dev->child, gh.ch->data(), L1 * sizeof(void *), cudaMemcpyHostToDevice));
    if (gh.id) {   // replica graphs: the tables the filtered search (hnsw_warp.cu) reads
        gh.id->assign(L1, nullptr); gh.md->assign(L1, nullptr);
        for (uint32_t L = 0; L < L1; ++L) { (*gh.id)[L] = st.g.lv[L].node_id; (*gh.md)[L] = st.g.lv[L].node_md; }
        CDB_CUDA_TRY(cudaMemcpy((void *)gh.id_tbl, gh.id->data(), L1 * sizeof(void *), cudaMemcpyHostToDevice));
        CDB_CUDA_TRY(cudaMemcpy((void *)gh.md_tbl, gh.md->data(), L1 * sizeof(void *), cudaMemcpyHostToDevice));
    }
    return CDB_OK;
}

cdb_status hnsw_build_smem_check(uint32_t row_pitch, uint32_t ef) {
    int dev = 0, optin = 0;
    CDB_CUDA_TRY(cudaGetDevice(&dev));
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const size_t need = hw_carve(row_pitch, ef).total;   // hnsw_build_search_kernel declares no static shared memory
    if (need > (size_t)optin) {
        set_error("hnsw build: ef " + std::to_string(ef) + " with " + std::to_string(row_pitch) + "-byte rows needs " +
                  std::to_string(need) + " bytes of shared memory per block, the device allows " + std::to_string(optin));
        return CDB_INVALID_PARAMS;
    }
    return CDB_OK;
}

// What an insert appends (planned before anything changes, so node_row / child are static while the adjacency evolves):
// per level the nodes' vector rows and, on levels >= 1, their children one level down; on replica graphs the nodes'
// columns; and the top level of each entry.
struct InsertPlan {
    std::vector<std::vector<uint32_t>> rows, child;
    ReplicaCols cols;
    std::vector<uint8_t> levels;
};

// rows [first, first + levels.size()) of a plain graph (levels[i] = max insert level of row first+i): level 0 holds node = row,
// levels >= 1 take ascending rows after the existing nodes, with child pointing into the appended part of the level below
static InsertPlan plan_rows(const HnswBuildState &st, uint32_t first, std::vector<uint8_t> levels, const uint32_t *h_deleted) {
    const uint32_t L1 = st.g.num_levels + 1, count = (uint32_t)levels.size();
    InsertPlan p;
    p.rows.resize(L1); p.child.resize(L1);
    for (uint32_t i = 0; h_deleted && i < count; ++i)   // a deleted row gets no upper-level nodes (and is not linked)
        if ((h_deleted[(first + i) >> 5] >> ((first + i) & 31)) & 1u) levels[i] = 0;
    for (uint32_t r = std::max(first, st.g.lv[0].cnt); r < first + count; ++r) p.rows[0].push_back(r);
    for (uint32_t i = 0; i < count; ++i)
        for (uint32_t L = 1; L <= levels[i]; ++L) p.rows[L].push_back(first + i);
    for (uint32_t L = 1; L < L1; ++L) {
        uint32_t j = 0;   // position in the rows appended one level down (both lists ascend)
        for (uint32_t r : p.rows[L]) {
            if (L == 1) { p.child[L].push_back(r); continue; }
            while (p.rows[L - 1][j] != r) ++j;
            p.child[L].push_back(st.g.lv[L - 1].cnt + j);
        }
    }
    p.levels = std::move(levels);
    return p;
}

// the entries of `rh` on a replica graph: list positions continue from st.n_list, new nodes follow the existing ones on every
// level they reach in list order, children at their position among the nodes appended one level down
static InsertPlan plan_replicas(const HnswBuildState &st, const ReplicaHost &rh) {
    const uint32_t L1 = st.g.num_levels + 1, n = rh.n_nodes;
    InsertPlan p;
    p.rows.resize(L1); p.child.resize(L1);
    p.cols.id.resize(L1); p.cols.md.resize(L1); p.cols.ins.resize(L1);
    p.levels.resize(n);
    std::vector<std::vector<uint32_t>> members(L1);   // new list indices present on each level
    for (uint32_t t = 0; t < n; ++t) {
        p.levels[t] = (uint8_t)std::min<uint32_t>(rh.max_level[t], st.g.num_levels);
        for (uint32_t L = 0; L <= p.levels[t]; ++L) {
            members[L].push_back(t);
            p.rows[L].push_back(rh.row[t]);
            p.cols.id[L].push_back(rh.node_id[t]);
            p.cols.md[L].push_back(rh.md_row[t]);
            p.cols.ins[L].push_back(st.n_list + t);
        }
    }
    for (uint32_t L = 1; L < L1; ++L) {
        uint32_t j = 0;   // position among the nodes appended one level down (both lists ascend)
        for (uint32_t t : members[L]) {
            while (members[L - 1][j] != t) ++j;
            p.child[L].push_back(st.g.lv[L - 1].cnt + j);
        }
    }
    return p;
}

// the Metadata table and the edge rules' keys of a replica graph (rows and ids are the caller's)
static ReplicaDev replica_table(const int32_t *md_bits, const float *md_mags, uint32_t M) {
    ReplicaDev rl{};
    rl.md_bits = md_bits;
    rl.md_mags = md_mags;
    rl.M = M;
    rl.key_one = order_key(CDB_METRIC_COSINE, 0x3F800000u);
    rl.key_minus_one = order_key(CDB_METRIC_COSINE, 0xBF800000u);
    return rl;
}

// index_embeddings for the planned entries [first, first + count) (rows, or on replica graphs list positions with `rl` indexed
// by them), the one batch loop of the build, the insert and their replica forms.  The planned nodes are appended up front.
// Batches hold max(1, min(max_batch, (linked + done) / 8)) entries, linked = entries already in the graph: a fresh build starts
// almost sequentially, a small transaction into a large graph runs as one batch.  Every allocation happens before the graph
// changes; *changed tells the caller whether an error left it half-inserted.
static cdb_status insert_planned(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState &st, const InsertPlan &p, uint32_t first,
                                 uint32_t linked, uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint64_t rows_cap,
                                 uint8_t *out_failed, bool *changed, cudaStream_t s, const uint32_t *d_deleted, const ReplicaDev *rl,
                                 const char *what) {
    const uint32_t L1 = st.g.num_levels + 1, count = (uint32_t)p.levels.size();
    cdb_status rc;
    if (max_batch == 0) max_batch = 4096;
    max_batch = std::max<uint32_t>(1, std::min(max_batch, count));
    DevAllocs tmp;
    uint8_t *d_levels = nullptr, *failed = nullptr;
    uint32_t *z_nodes = nullptr, *z_keys = nullptr, *z_n = nullptr;
    if ((rc = tmp.get((void **)&d_levels, count)) || (rc = tmp.get((void **)&failed, count)) ||
        (rc = tmp.get((void **)&z_nodes, (size_t)max_batch * L1 * 64 * 4)) || (rc = tmp.get((void **)&z_keys, (size_t)max_batch * L1 * 64 * 4)) ||
        (rc = tmp.get((void **)&z_n, (size_t)max_batch * L1 * 4)))
        return rc;
    const HwCarve cv = hw_carve(sc.row_pitch, ef_construction);
    const BuildSearchKernel search = build_search_kernel(sc, rl != nullptr);
    CDB_ALLOW_SMEM(search, cv.total);
    if ((rc = append_levels(st, gh, p.rows, p.child, rows_cap, changed, s, rl ? &p.cols : nullptr))) return rc;
    if (!count) return CDB_OK;
    // ---- batches
    CDB_CUDA_TRY(cudaMemcpyAsync(d_levels, p.levels.data(), count, cudaMemcpyHostToDevice, s));
    BuildArgs a{};
    a.g = st.g;
    a.sc = sc;
    a.sc.root_row = st.g.root_row;
    a.levels = d_levels;
    a.lv_first = first;
    a.ef = ef_construction;
    a.shortlist = shortlist;
    a.zcap = 64;
    a.z_nodes = z_nodes; a.z_keys = z_keys; a.z_n = z_n;
    a.deleted = d_deleted;
    a.replicas = rl != nullptr;
    if (rl) a.rl = *rl;
    for (uint32_t done = 0; done < count;) {
        uint32_t batch = std::max<uint32_t>(1, std::min<uint32_t>(max_batch, (uint32_t)(((uint64_t)linked + done) / 8)));
        batch = std::min<uint32_t>(batch, count - done);
        a.first = first + done;
        a.count = batch;
        a.failed = failed + done;
        search<<<batch, 32, cv.total, s>>>(a, cv);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        hnsw_build_link_kernel<<<(batch * 32 + 127) / 128, 128, 0, s>>>(a);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        done += batch;
    }
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e == cudaSuccess && out_failed) e = cudaMemcpy(out_failed, failed, count, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { set_error(std::string(what) + ": " + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    return CDB_OK;
}

// a fresh builder state for a graph of num_levels + 1 empty levels, and the search layout's pointer tables; the roots are
// appended next
static cdb_status new_graph(int metric, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0, uint32_t root_row, uint32_t entry,
                            uint32_t identity_mask, const GraphHost &gh, std::unique_ptr<HnswBuildState> &st) {
    if (num_levels + 1 > BUILD_MAX_LEVELS) { set_error("build: too many levels"); return CDB_INVALID_PARAMS; }
    const uint32_t L1 = num_levels + 1;
    st.reset(new HnswBuildState());
    st->g.num_levels = num_levels;
    st->g.root_row = root_row;
    st->g.entry = entry;
    metric_key_range(metric, &st->g.min_key, &st->g.max_key);
    for (uint32_t L = 0; L < L1; ++L) st->g.lv[L].nb = L == 0 ? nbrs0 : nbrs;
    const uint32_t *tbl[3];
    for (int t = 0; t < 3; ++t) {
        void *p = nullptr;
        CDB_CUDA_TRY(cudaMalloc(&p, L1 * sizeof(void *)));
        gh.allocs->push_back(p);
        tbl[t] = (const uint32_t *)p;
    }
    gh.dev->num_levels = num_levels;
    gh.dev->nbrs = nbrs;
    gh.dev->nbrs0 = nbrs0;
    gh.dev->entry = entry;
    gh.dev->root_row = root_row;
    gh.dev->identity_mask = identity_mask;
    gh.dev->node_row = reinterpret_cast<const uint32_t *const *>(tbl[0]);
    gh.dev->adj = reinterpret_cast<const uint32_t *const *>(tbl[1]);
    gh.dev->child = reinterpret_cast<const uint32_t *const *>(tbl[2]);
    return CDB_OK;
}

cdb_status hnsw_build_device(const HnScoreCtx &sc, uint32_t n /* data rows; root is row n */, uint32_t num_levels, uint32_t nbrs,
                             uint32_t nbrs0, uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint64_t seed,
                             const GraphHost &gh, HnswBuildState **out_state, cudaStream_t s, const uint32_t *d_deleted,
                             const uint32_t *h_deleted) {
    // level 0: node i is row i (lv_local), the search skips the node_row lookup there
    std::unique_ptr<HnswBuildState> st;
    cdb_status rc = new_graph(sc.metric, num_levels, nbrs, nbrs0, n, num_levels == 0 ? n : 0, 1u, gh, st);
    if (rc) return rc;
    // ---- the root on every level (vector_store.rs:44-140); level 0 holds a node for every row, linked once inserted
    const uint32_t L1 = num_levels + 1;
    bool changed = false;
    std::vector<std::vector<uint32_t>> rows(L1), child(L1);
    for (uint32_t i = 0; i <= n; ++i) rows[0].push_back(i);
    for (uint32_t L = 1; L < L1; ++L) { rows[L] = {n}; child[L] = {L == 1 ? n : 0u}; }
    if ((rc = append_levels(*st, gh, rows, child, n + 1, &changed, s))) return rc;
    // ---- then every data row through the insert path
    std::vector<uint8_t> levels(n);
    for (uint32_t r = 0; r < n; ++r) levels[r] = draw_level(seed, r, num_levels);
    rc = insert_planned(sc, gh, *st, plan_rows(*st, 0, std::move(levels), h_deleted), 0, 0, ef_construction, shortlist, max_batch, n + 1,
                        nullptr, &changed, s, d_deleted, nullptr, "hnsw build");
    if (rc) return rc;
    *out_state = st.release();
    return CDB_OK;
}

cdb_status hnsw_insert_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, uint32_t n_new, const uint8_t *max_level,
                              uint64_t seed, uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint64_t rows_cap,
                              uint8_t *out_failed, bool *changed, cudaStream_t s, const uint32_t *d_deleted, const uint32_t *h_deleted) {
    const uint32_t first = (*gh.cnt)[0], num_levels = st->g.num_levels;   // the published graph
    std::vector<uint8_t> levels(n_new);
    for (uint32_t i = 0; i < n_new; ++i)
        levels[i] = max_level ? (uint8_t)std::min<uint32_t>(max_level[i], num_levels) : draw_level(seed, first + i, num_levels);
    return insert_planned(sc, gh, *st, plan_rows(*st, first, std::move(levels), h_deleted), first, first - 1, ef_construction, shortlist,
                          max_batch, rows_cap, out_failed, changed, s, d_deleted, nullptr, "hnsw build");
}

cdb_status hnsw_slot_state_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState **out_state, cudaStream_t s) {
    const GraphDev &d = *gh.dev;
    const uint32_t L1 = d.num_levels + 1;
    if (L1 > BUILD_MAX_LEVELS) { set_error("the graph has more levels than the builder supports"); return CDB_UNSUPPORTED; }
    const uint32_t rows_fit = SS_STAGE_BYTES / sc.row_pitch;   // node row + `group` neighbour rows per warp
    const uint32_t group = rows_fit >= 2 ? std::min<uint32_t>(32, rows_fit - 1) : 1u;
    const size_t smem = (size_t)SS_WARPS * (group + 1) * sc.row_pitch;
    int dev = 0, optin = 0;
    CDB_CUDA_TRY(cudaGetDevice(&dev));
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if (smem + SS_WARPS * 8 > (size_t)optin) { set_error("slot state: rows too wide for shared memory"); return CDB_UNSUPPORTED; }
    CDB_ALLOW_SMEM(hnsw_slot_state_kernel, smem);
    std::unique_ptr<HnswBuildState> st(new HnswBuildState());
    st->g.num_levels = d.num_levels;
    st->g.entry = d.entry;
    st->g.root_row = d.root_row;
    metric_key_range(sc.metric, &st->g.min_key, &st->g.max_key);
    HnScoreCtx c = sc;
    c.root_row = d.root_row;
    for (uint32_t L = 0; L < L1; ++L) {
        BuildLevel &l = st->g.lv[L];
        l.cnt = l.app = (*gh.cnt)[L];
        l.nb = L == 0 ? d.nbrs0 : d.nbrs;
        l.node_row = const_cast<uint32_t *>((*gh.nr)[L]);
        l.adj = const_cast<uint32_t *>((*gh.ad)[L]);
        l.child = L ? const_cast<uint32_t *>((*gh.ch)[L]) : nullptr;
        st->cap[L] = l.cnt;
        void *p[4];
        const size_t words[4] = {(size_t)l.cnt * l.nb, l.cnt, l.cnt, l.cnt};
        for (int t = 0; t < 4; ++t) {
            CDB_CUDA_TRY(cudaMalloc(&p[t], std::max<size_t>(words[t], 1) * 4));
            gh.allocs->push_back(p[t]);
        }
        l.simkey = (uint32_t *)p[0]; l.lowest_idx = (uint32_t *)p[1]; l.lowest_key = (uint32_t *)p[2]; l.lock = (int *)p[3];
        CDB_CUDA_TRY(cudaMemsetAsync(l.simkey, 0, words[0] * 4, s));
        CDB_CUDA_TRY(cudaMemsetAsync(l.lock, 0, (size_t)l.cnt * 4, s));
        if (!l.cnt) continue;
        const uint32_t grid = (l.cnt + SS_WARPS - 1) / SS_WARPS;
        hnsw_slot_state_kernel<<<grid, SS_WARPS * 32, smem, s>>>(l, c, st->g.min_key, st->g.max_key, group);
        CDB_LAUNCH_CHECK();
    }
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error(std::string("hnsw slot state: ") + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    *out_state = st.release();
    return CDB_OK;
}

// ------------------------------------------------------------------ delete_embedding (vector_store.rs:1206-1371)
// Phase A is hnsw_build_search_kernel in delete mode (rowlist set: nothing pre-seeded, ef 512, best 100 kept).  Phase B runs
// one warp per (delete, level): remove_neighbor_by_id on each neighbour in D's slot order, relink a neighbour that emptied
// (create_node_edges over the results, rescored against it), then clear D's slots.  The sweep then clears every remaining
// slot that names a node deleted in the batch (D2), and the nodes it touched are relinked if empty at their turn, in
// ascending level-local index when deletes run one at a time.  A level's repair never reads or writes another level.
struct DelArgs {
    BuildGraph g;
    HnScoreCtx sc;
    // the batch positions are items: the deleted rows on a plain graph, every node of a deleted row on a replica graph; the
    // batch's rows own items [row_items[j], row_items[j+1]) for j from rfirst
    const uint32_t *loc;    // [items][num_levels+1] level-local index of each item (HN_EMPTY: not on that level)
    uint32_t first, count, zcap;
    const uint32_t *z_nodes, *z_n;
    uint8_t *status;        // [items] 2 where a rescoring Err stopped a relink
    uint32_t *dead[BUILD_MAX_LEVELS];      // [cnt/32+1] nodes deleted by this call
    uint32_t *dead_of[BUILD_MAX_LEVELS];   // [cnt] batch position of a deleted node
    uint32_t *touched[BUILD_MAX_LEVELS];   // [cnt/32+1] nodes the sweep cleared a slot of
    uint2 *list[BUILD_MAX_LEVELS];         // [cnt] (node, batch position) of each touched node
    uint32_t *list_n;                      // [num_levels+1]
    // replica graphs (hnsw_delete_replicas_device): relinks rescore with the replica arms and apply the edge rules, and a
    // touched node takes the candidates of the smallest batch position it named (tmin)
    bool replicas;
    ReplicaDev rl;                         // the Metadata table and the edge rules' keys
    const uint32_t *row_items;
    uint32_t rfirst;
    uint32_t *tmin[BUILD_MAX_LEVELS];      // [cnt] HN_EMPTY between calls; null on plain graphs
};

__global__ void hnsw_delete_mark_kernel(DelArgs a) {
    const uint32_t L1 = a.g.num_levels + 1;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < L1) a.list_n[t] = 0;
    if (t >= a.count * L1) return;
    const uint32_t b = t / L1, L = t % L1, D = a.loc[(size_t)(a.first + b) * L1 + L];
    if (D == HN_EMPTY) return;
    atomicOr(a.dead[L] + (D >> 5), 1u << (D & 31));
    a.dead_of[L][D] = b;
}

// remove_neighbor_by_id (prob_node.rs:285-306): the first slot naming `id` is cleared, lowest_index is left stale
__device__ bool build_remove_by_id(const BuildLevel &l, uint32_t node, uint32_t id) {
    volatile uint32_t *na = l.adj + (size_t)node * l.nb;
    bool found = false;
    node_lock(l.lock + node);
    for (uint32_t s = 0; s < l.nb && !found; ++s)
        if (na[s] == id) { na[s] = HN_EMPTY; found = true; }
    node_unlock(l.lock + node);
    return found;
}
__device__ bool build_is_empty(const BuildLevel &l, uint32_t node) {
    const volatile uint32_t *na = l.adj + (size_t)node * l.nb;
    for (uint32_t s = 0; s < l.nb; ++s)
        if (na[s] != HN_EMPTY) return false;
    return true;
}

// one side of calculate() for a node of a replica graph: VectorData { Some(get_id()), vector, metadata }
__device__ __forceinline__ MdSide del_md_side(const ReplicaDev &rl, const BuildLevel &l, uint32_t node, const void *code, float mag,
                                              uint32_t pp) {
    const uint32_t mrow = l.node_md[node];
    return MdSide{code, mag, pp, true, l.node_id[node], mrow == HN_EMPTY ? nullptr : rl.md_bits + (size_t)mrow * rl.M,
                  mrow == HN_EMPTY ? 0.0f : rl.md_mags[mrow]};
}

struct DelSmem {
    uint64_t keys[2][128];
    uint32_t nodes[2][128];
    uint64_t bar;
};

// The relink of an emptied node N (vector_store.rs:1306-1357), whole warp: the results minus D, N and the nodes this call
// deletes are rescored against N (N's row staged by one bulk copy, candidates scored one per lane with pair_distance), sorted
// best first (ties: smaller id), then lane 0 runs create_node_edges with N's stale lowest_index.  false: a rescoring Err.
__device__ bool del_relink(const DelArgs &a, uint32_t level, uint32_t N, uint32_t D, const uint32_t *cand, uint32_t zn, uint8_t *row,
                           DelSmem &sm, uint32_t &parity) {
    const BuildLevel &l = a.g.lv[level];
    const HnScoreCtx &sc = a.sc;
    const uint32_t lane = threadIdx.x & 31, bar = hw_smem_u32(&sm.bar);
    const uint32_t nrow = l.node_row[N];
    const bool rules = a.replicas && sc.metric == CDB_METRIC_COSINE;   // the rules match MetricResult::CosineSimilarity only
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    if (lane == 0) {
        hw_mbar_expect(bar, sc.row_pitch);
        hw_bulk_g2s(hw_smem_u32(row), sc.rows + (size_t)nrow * sc.row_pitch, sc.row_pitch, bar);
    }
    hw_mbar_wait(bar, parity);
    parity ^= 1u;
    const uint32_t pp = plane_pitch(sc.dim);
    uint32_t m = 0;
    bool bad = false;
    for (uint32_t base = 0; base < zn; base += 32) {
        const uint32_t i = base + lane;
        const uint32_t c = i < zn ? cand[i] : HN_EMPTY;
        const bool keep = c != HN_EMPTY && c != D && c != N && !bit_set(a.dead[level], c);
        const uint32_t ball = __ballot_sync(0xFFFFFFFFu, keep);
        if (keep) {
            const uint32_t crow = l.node_row[c], pos = m + __popc(ball & ((1u << lane) - 1u));
            const uint8_t *ccode = sc.rows + (size_t)crow * sc.row_pitch;
            float d = 0.f;
            int rc;
            uint32_t cid;
            if (a.replicas) {   // calculate(N, cand) with the replica arms: N's id and metadata are x
                rc = md_pair_distance(sc.metric, sc.st, sc.dim, a.rl.M, del_md_side(a.rl, l, N, row, sc.mags[nrow], pp),
                                      del_md_side(a.rl, l, c, ccode, sc.mags[crow], pp), &d);
                cid = l.node_id[c];
            } else {
                rc = pair_distance(sc.metric, sc.st, sc.dim, row, sc.mags[nrow], pp, ccode, sc.mags[crow], pp, &d);
                cid = hn_id(sc.root_row, crow);
            }
            if (rc != CDB_OK) bad = true;
            sm.keys[0][pos] = make_key64(order_key(sc.metric, __float_as_uint(d)), cid);
            sm.nodes[0][pos] = c;
        }
        m += __popc(ball);
    }
    if (__any_sync(0xFFFFFFFFu, bad)) return false;
    __syncwarp();
    for (uint32_t i = lane; i < m; i += 32) {   // rank sort, best first (keys are unique: one per node)
        const uint64_t k = sm.keys[0][i];
        uint32_t r = 0;
        for (uint32_t j = 0; j < m; ++j) r += sm.keys[0][j] > k;
        sm.keys[1][r] = k;
        sm.nodes[1][r] = sm.nodes[0][i];
    }
    __syncwarp();
    if (lane == 0) {   // create_node_edges (vector_store.rs:976-1070); on replica graphs with the rules of :1014-1040
        const int nk = rules ? build_node_kind(a.rl, l, N) : MD_KIND_BASE;
        uint32_t successful = 0;
        for (uint32_t i = 0; i < m; ++i) {
            if (successful >= l.nb) break;
            const uint32_t nbr = sm.nodes[1][i], dkey = (uint32_t)(sm.keys[1][i] >> 32);
            if (nk == MD_KIND_METADATA) {   // as hnsw_build_link_kernel
                const int bk = build_node_kind(a.rl, l, nbr);
                if (bk == MD_KIND_PSEUDO && dkey != a.rl.key_one) continue;
                if (bk == MD_KIND_METADATA && dkey == a.rl.key_minus_one) continue;
            }
            const int idx = build_add_neighbor(a.g, l, N, nbr, dkey);
            if (idx < 0) continue;
            if (build_add_neighbor(a.g, l, nbr, N, dkey) >= 0) { successful++; continue; }
            volatile uint32_t *na = l.adj + (size_t)N * l.nb;
            node_lock(l.lock + N);
            if (na[idx] == nbr) na[idx] = HN_EMPTY;
            node_unlock(l.lock + N);
        }
    }
    __syncwarp();
    return true;
}

__device__ inline void del_smem_init(DelSmem &sm) {
    if ((threadIdx.x & 31) == 0) hw_mbar_init(hw_smem_u32(&sm.bar), 1);
    __syncwarp();
}

// phase B for the node D of batch position b on `level` (whole warp): D's own slots, then D isolated
__device__ void del_repair_node(const DelArgs &a, uint32_t level, uint32_t b, uint32_t D, uint8_t *row, DelSmem &sm, uint32_t &parity) {
    const uint32_t L1 = a.g.num_levels + 1, lane = threadIdx.x & 31;
    const BuildLevel &l = a.g.lv[level];
    const uint32_t zn = a.z_n[(size_t)b * L1 + level];
    const uint32_t *cand = a.z_nodes + ((size_t)b * L1 + level) * a.zcap;
    bool err = false;
    volatile uint32_t *da = l.adj + (size_t)D * l.nb;
    for (uint32_t s = 0; s < l.nb; ++s) {
        uint32_t N = lane == 0 ? da[s] : 0u;
        N = __shfl_sync(0xFFFFFFFFu, N, 0);
        if (N == HN_EMPTY) continue;
        int go = 0;
        if (lane == 0) go = build_remove_by_id(l, N, D) && !bit_set(a.dead[level], N) && build_is_empty(l, N);
        go = __shfl_sync(0xFFFFFFFFu, go, 0);
        if (go && zn != HN_EMPTY && !del_relink(a, level, N, D, cand, zn, row, sm, parity)) err = true;
    }
    if (lane == 0) {   // D4: the node stays, isolated
        node_lock(l.lock + D);
        for (uint32_t s = 0; s < l.nb; ++s) da[s] = HN_EMPTY;
        ((volatile uint32_t *)l.lowest_idx)[D] = 0;
        ((volatile uint32_t *)l.lowest_key)[D] = a.g.min_key;
        node_unlock(l.lock + D);
        if (err) a.status[a.first + b] = 2;
    }
    __syncwarp();
}

// phase B: one warp (one block) per (deleted row, level) repairs the row's items on that level in order -- on a replica graph
// two replicas of a row can share neighbours, so one after the other keeps the result deterministic; on a plain graph a row
// is one item
__global__ void __launch_bounds__(32) hnsw_delete_repair_kernel(DelArgs a) {
    extern __shared__ __align__(128) uint8_t row[];
    __shared__ DelSmem sm;
    const uint32_t L1 = a.g.num_levels + 1, j = a.rfirst + blockIdx.x / L1, level = blockIdx.x % L1;
    del_smem_init(sm);
    uint32_t parity = 0;
    for (uint32_t k = a.row_items[j]; k < a.row_items[j + 1]; ++k) {
        const uint32_t D = a.loc[(size_t)k * L1 + level];
        if (D != HN_EMPTY) del_repair_node(a, level, k - a.first, D, row, sm, parity);
    }
}

// D2: one pass over the level's adjacency (128-bit loads, grid-stride) clears every slot naming a node deleted by this call
// and lists each node it cleared a slot of once, with the batch position of (one of) the deleted nodes it named
__device__ __forceinline__ bool del_sweep_slot(const DelArgs &a, uint32_t level, uint64_t t, uint32_t &v) {
    if (v == HN_EMPTY || !bit_set(a.dead[level], v)) return false;
    const uint32_t node = (uint32_t)(t / a.g.lv[level].nb), bit = 1u << (node & 31);
    if (!(atomicOr(a.touched[level] + (node >> 5), bit) & bit))
        a.list[level][atomicAdd(a.list_n + level, 1u)] = make_uint2(node, a.dead_of[level][v]);
    if (a.tmin[level]) atomicMin(a.tmin[level] + node, a.dead_of[level][v]);   // replica graphs: the smallest position named
    v = HN_EMPTY;
    return true;
}
__global__ void hnsw_delete_sweep_kernel(DelArgs a, uint32_t level) {
    const BuildLevel &l = a.g.lv[level];
    const uint64_t slots = (uint64_t)l.cnt * l.nb, vecs = slots / 4;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    uint4 *adj4 = reinterpret_cast<uint4 *>(l.adj);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < vecs; i += stride) {
        uint4 v = adj4[i];
        bool ch = del_sweep_slot(a, level, 4 * i, v.x);
        ch |= del_sweep_slot(a, level, 4 * i + 1, v.y);
        ch |= del_sweep_slot(a, level, 4 * i + 2, v.z);
        ch |= del_sweep_slot(a, level, 4 * i + 3, v.w);
        if (ch) adj4[i] = v;
    }
    const uint64_t t = vecs * 4 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < slots) {
        uint32_t v = l.adj[t];
        if (del_sweep_slot(a, level, t, v)) l.adj[t] = v;
    }
}

// relink of the nodes the sweep touched: one warp per list entry, or (ordered, deletes one at a time) a single warp taking
// the entries in ascending node index.  A node is relinked if it is empty at its turn and not deleted itself.
__global__ void __launch_bounds__(32) hnsw_delete_relink_kernel(DelArgs a, uint32_t level, bool ordered) {
    extern __shared__ __align__(128) uint8_t row[];
    __shared__ DelSmem sm;
    const uint32_t L1 = a.g.num_levels + 1, lane = threadIdx.x & 31, n = a.list_n[level];
    if (!n) return;
    del_smem_init(sm);
    const BuildLevel &l = a.g.lv[level];
    const uint2 *list = a.list[level];
    uint32_t parity = 0;
    uint32_t *tmin = a.tmin[level];
    auto process = [&](uint2 e) {
        const uint32_t X = e.x, b = tmin ? tmin[X] : e.y;
        const uint32_t zn = a.z_n[(size_t)b * L1 + level];
        int go = 0;
        if (lane == 0) go = zn != HN_EMPTY && !bit_set(a.dead[level], X) && build_is_empty(l, X);
        if (!__shfl_sync(0xFFFFFFFFu, go, 0)) return;
        const uint32_t D = a.loc[(size_t)(a.first + b) * L1 + level];
        if (!del_relink(a, level, X, D, a.z_nodes + ((size_t)b * L1 + level) * a.zcap, zn, row, sm, parity) && lane == 0)
            a.status[a.first + b] = 2;
    };
    if (!ordered) {
        for (uint32_t e = blockIdx.x; e < n; e += gridDim.x) {
            process(list[e]);
            if (lane == 0) atomicAnd(a.touched[level] + (list[e].x >> 5), ~(1u << (list[e].x & 31)));
            if (lane == 0 && tmin) tmin[list[e].x] = HN_EMPTY;
        }
        return;
    }
    if (blockIdx.x) return;
    int64_t last = -1;
    for (;;) {
        uint64_t best = ~0ull;   // (node << 32 | entry) of the smallest node above `last`
        for (uint32_t e = lane; e < n; e += 32)
            if ((int64_t)list[e].x > last) best = min(best, ((uint64_t)list[e].x << 32) | e);
        for (int o = 16; o; o >>= 1) best = min(best, (uint64_t)__shfl_xor_sync(0xFFFFFFFFu, best, o));
        if (best == ~0ull) break;
        last = (int64_t)(best >> 32);
        process(list[(uint32_t)best]);
    }
    for (uint32_t e = lane; e < n; e += 32) {
        atomicAnd(a.touched[level] + (list[e].x >> 5), ~(1u << (list[e].x & 31)));
        if (tmin) tmin[list[e].x] = HN_EMPTY;
    }
}

// The nodes a delete repairs, as items grouped by row: each item's level-local index per level, what phase A traverses, and
// the index in the call of the row each item belongs to.  Plain graphs: one item per row with a level-0 node, traversed as
// that row.  Replica graphs: every node of a deleted row, traversed as the per-item columns.
struct DelItems {
    std::vector<uint32_t> loc;         // [items][num_levels+1]
    std::vector<uint32_t> row_items;   // [rows + 1] the items of the j-th row with items are [row_items[j], row_items[j+1])
    std::vector<uint32_t> rowlist;     // [items] plain: the item's row; replica: 0..items-1, indexing `cols`
    std::vector<uint32_t> cols;        // replica graphs: [3][items] vector row, node_id, Metadata row
    std::vector<uint32_t> out;         // [items] index in the call of the item's row
};

// delete_embedding for the items (none empty), the one batch loop of both deletes: per batch of max_batch rows the mark, phase
// A over the batch's items, the repair of each (row, level), then per level the sweep and the relink.  out_status[out[k]] = 2
// where an Err hit item k.  Every allocation happens before the graph changes; *changed as for the insert.
static cdb_status delete_items(const HnScoreCtx &sc, HnswBuildState *st, const DelItems &it, uint32_t shortlist, uint32_t max_batch,
                               uint8_t *out_status, bool *changed, cudaStream_t s, int sms, const char *what) {
    const uint32_t L1 = st->g.num_levels + 1, ni = (uint32_t)it.rowlist.size(), ng = (uint32_t)it.row_items.size() - 1;
    const bool replicas = st->replicas;
    constexpr uint32_t DEL_EF = HNSW_DELETE_EF, DEL_KEEP = 100;   // the reference's literal ef and final_len (vector_store.rs:1194, 1247)
    if (max_batch == 0) max_batch = 4096;
    max_batch = std::max<uint32_t>(1, std::min(max_batch, ng));
    uint32_t max_items = 0;
    for (uint32_t j = 0; j < ng; j += max_batch)
        max_items = std::max(max_items, it.row_items[std::min(ng, j + max_batch)] - it.row_items[j]);
    // ---- every allocation before the graph changes
    cdb_status rc;
    DevAllocs tmp;
    DelArgs d{};
    uint32_t *d_rowlist = nullptr, *d_cols = nullptr, *d_loc = nullptr, *d_ri = nullptr, *z_nodes = nullptr, *z_keys = nullptr, *z_n = nullptr;
    uint8_t *failed = nullptr;
    if ((rc = tmp.get((void **)&d_rowlist, (size_t)ni * 4)) || (replicas && (rc = tmp.get((void **)&d_cols, it.cols.size() * 4))) ||
        (rc = tmp.get((void **)&d_loc, it.loc.size() * 4)) || (rc = tmp.get((void **)&d_ri, it.row_items.size() * 4)) ||
        (rc = tmp.get((void **)&z_nodes, (size_t)max_items * L1 * DEL_KEEP * 4)) ||
        (rc = tmp.get((void **)&z_keys, (size_t)max_items * L1 * DEL_KEEP * 4)) || (rc = tmp.get((void **)&z_n, (size_t)max_items * L1 * 4)) ||
        (rc = tmp.get((void **)&failed, ni)) || (rc = tmp.get((void **)&d.status, ni)) || (rc = tmp.get((void **)&d.list_n, L1 * 4)))
        return rc;
    for (uint32_t L = 0; L < L1; ++L) {
        const uint32_t cnt = st->g.lv[L].cnt, words = cnt / 32 + 1;
        if ((rc = tmp.get((void **)&d.dead[L], (size_t)words * 4)) || (rc = tmp.get((void **)&d.touched[L], (size_t)words * 4)) ||
            (rc = tmp.get((void **)&d.dead_of[L], (size_t)cnt * 4)) || (rc = tmp.get((void **)&d.list[L], (size_t)cnt * 8)) ||
            (replicas && (rc = tmp.get((void **)&d.tmin[L], (size_t)cnt * 4))))
            return rc;
        CDB_CUDA_TRY(cudaMemsetAsync(d.dead[L], 0, (size_t)words * 4, s));
        CDB_CUDA_TRY(cudaMemsetAsync(d.touched[L], 0, (size_t)words * 4, s));
        if (replicas) CDB_CUDA_TRY(cudaMemsetAsync(d.tmin[L], 0xFF, (size_t)cnt * 4, s));
    }
    const HwCarve cv = hw_carve(sc.row_pitch, DEL_EF);
    const BuildSearchKernel search = build_search_kernel(sc, replicas);
    CDB_ALLOW_SMEM(search, cv.total);
    CDB_ALLOW_SMEM(hnsw_delete_repair_kernel, sc.row_pitch);
    CDB_ALLOW_SMEM(hnsw_delete_relink_kernel, sc.row_pitch);
    CDB_CUDA_TRY(cudaMemsetAsync(d.status, 0, ni, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(d_rowlist, it.rowlist.data(), (size_t)ni * 4, cudaMemcpyHostToDevice, s));
    if (replicas) CDB_CUDA_TRY(cudaMemcpyAsync(d_cols, it.cols.data(), it.cols.size() * 4, cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(d_loc, it.loc.data(), it.loc.size() * 4, cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaMemcpyAsync(d_ri, it.row_items.data(), it.row_items.size() * 4, cudaMemcpyHostToDevice, s));
    // ---- batches of rows
    *changed = true;
    BuildArgs a{};
    a.g = st->g;
    a.sc = sc;
    a.sc.root_row = st->g.root_row;
    a.ef = DEL_EF;
    a.shortlist = shortlist;
    a.zcap = DEL_KEEP;
    a.z_nodes = z_nodes; a.z_keys = z_keys; a.z_n = z_n;
    a.rowlist = d_rowlist;
    a.replicas = replicas;
    if (replicas) {
        // the traversal of an item carries Some(its node_id) as the query id; that id only decides the Pseudo kind
        // (types.rs:232), which a data row's replicas never have (the pseudo root's row cannot be deleted)
        a.rl = replica_table(st->md_bits, st->md_mags, st->md_dims);
        a.rl.row = d_cols;
        a.rl.id = d_cols + ni;
        a.rl.base_id = d_cols + ni;
        a.rl.md = d_cols + 2 * (size_t)ni;
    }
    d.g = st->g;
    d.sc = a.sc;
    d.loc = d_loc;
    d.zcap = DEL_KEEP;
    d.z_nodes = z_nodes; d.z_n = z_n;
    d.replicas = replicas;
    d.rl = a.rl;
    d.row_items = d_ri;
    const bool ordered = max_batch == 1;
    for (uint32_t rdone = 0; rdone < ng;) {
        const uint32_t rb = std::min(max_batch, ng - rdone), first = it.row_items[rdone], count = it.row_items[rdone + rb] - first;
        a.first = d.first = first;
        a.count = d.count = count;
        a.failed = failed + first;
        d.rfirst = rdone;
        hnsw_delete_mark_kernel<<<(count * L1 + 127) / 128, 128, 0, s>>>(d);
        search<<<count, 32, cv.total, s>>>(a, cv);
        hnsw_delete_repair_kernel<<<rb * L1, 32, sc.row_pitch, s>>>(d);
        g_launch_count.fetch_add(3, std::memory_order_relaxed);
        for (uint32_t L = 0; L < L1; ++L) {
            const uint64_t vecs = (uint64_t)a.g.lv[L].cnt * a.g.lv[L].nb / 4 + 1;
            const uint32_t grid = (uint32_t)std::min<uint64_t>((vecs + 255) / 256, (uint64_t)sms * 8);
            hnsw_delete_sweep_kernel<<<grid, 256, 0, s>>>(d, L);
            hnsw_delete_relink_kernel<<<ordered ? 1 : 1024, 32, sc.row_pitch, s>>>(d, L, ordered);
            g_launch_count.fetch_add(2, std::memory_order_relaxed);
        }
        rdone += rb;
    }
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    std::vector<uint8_t> hf(ni), hs(ni);
    if (e == cudaSuccess) e = cudaMemcpy(hf.data(), failed, ni, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(hs.data(), d.status, ni, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { set_error(std::string(what) + ": " + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    for (uint32_t k = 0; k < ni; ++k)
        if (hf[k] || hs[k]) out_status[it.out[k]] = 2;
    return CDB_OK;
}

static cdb_status sm_count(int *sms) {
    int dev = 0;
    CDB_CUDA_TRY(cudaGetDevice(&dev));
    CDB_CUDA_TRY(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
    return CDB_OK;
}

cdb_status hnsw_delete_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, const uint32_t *rows, uint32_t n,
                              uint32_t shortlist, uint32_t max_batch, uint8_t *out_status, bool *changed, cudaStream_t s) {
    const uint32_t L1 = st->g.num_levels + 1;
    // level-local index of every row on every level (level 0 is the row when the level lists rows in order)
    std::vector<uint32_t> loc((size_t)n * L1, HN_EMPTY);
    std::unordered_map<uint32_t, uint32_t> pos;
    for (uint32_t i = 0; i < n; ++i) pos.emplace(rows[i], i);
    for (uint32_t L = 0; L < L1; ++L) {
        const uint32_t cnt = (*gh.cnt)[L];
        if (L == 0 && (gh.dev->identity_mask & 1u)) {
            for (uint32_t i = 0; i < n; ++i) if (rows[i] < cnt) loc[(size_t)i * L1] = rows[i];
            continue;
        }
        std::vector<uint32_t> nr(cnt);
        if (cnt) CDB_CUDA_TRY(cudaMemcpy(nr.data(), (*gh.nr)[L], (size_t)cnt * 4, cudaMemcpyDeviceToHost));
        for (uint32_t j = 0; j < cnt; ++j) {
            auto it = pos.find(nr[j]);
            if (it != pos.end() && loc[(size_t)it->second * L1 + L] == HN_EMPTY) loc[(size_t)it->second * L1 + L] = j;
        }
    }
    // only rows with a level-0 node take part in the repair (a row appended after the graph was built is not in it)
    DelItems it;
    for (uint32_t i = 0; i < n; ++i) {
        out_status[i] = 0;
        if (loc[(size_t)i * L1] == HN_EMPTY) continue;
        it.row_items.push_back((uint32_t)it.out.size());
        it.out.push_back(i);
        it.rowlist.push_back(rows[i]);
        it.loc.insert(it.loc.end(), loc.begin() + (size_t)i * L1, loc.begin() + (size_t)(i + 1) * L1);
    }
    if (it.out.empty()) return CDB_OK;
    it.row_items.push_back((uint32_t)it.out.size());
    int sms = 0;
    cdb_status rc = sm_count(&sms);
    return rc ? rc : delete_items(sc, st, it, shortlist, max_batch, out_status, changed, s, sms, "hnsw delete");
}

// ------------------------------------------------------------------ replica lists (collections with a metadata schema)
// index_embeddings over the flattened IndexableEmbeddings (vector_store.rs:714-780): host arrays, one entry per node to create,
// into the replica graph of `st` behind the nodes earlier calls created.  Level layout: [0] main root, [1] pseudo root (both
// on every level, create_root_node / create_pseudo_root_node), then the created nodes in list order, with node_ins continuing
// the list positions, so build_local's binary search and both kernels run unchanged; ReplicaDev is offset so that it is indexed
// by those global positions.  Level draws come from the caller.  Every allocation (the list, the batch buffers, the grown
// Metadata table, the grown level arrays) happens before the graph changes; the table replaces the old one only once the
// insert has succeeded.
static cdb_status insert_replica_list(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState &st, const ReplicaHost &rh,
                                      uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint8_t *out_failed, bool *changed,
                                      cudaStream_t s, const char *what) {
    const uint32_t n = rh.n_nodes, first = st.n_list, M = st.md_dims;
    const InsertPlan p = plan_replicas(st, rh);
    cdb_status rc;
    DevAllocs tmp, table;
    uint32_t *d_list = nullptr;
    if ((rc = tmp.get((void **)&d_list, (size_t)n * 4 * 4))) return rc;
    const uint32_t n_md = st.n_md + rh.n_md;
    int32_t *new_bits = nullptr;
    float *new_mags = nullptr;
    if (rh.n_md) {   // the grown table: the old rows, then the new ones
        if ((rc = table.get((void **)&new_bits, (size_t)n_md * M * 4)) || (rc = table.get((void **)&new_mags, (size_t)n_md * 4))) return rc;
        if (st.n_md) {
            CDB_CUDA_TRY(cudaMemcpyAsync(new_bits, st.md_bits, (size_t)st.n_md * M * 4, cudaMemcpyDeviceToDevice, s));
            CDB_CUDA_TRY(cudaMemcpyAsync(new_mags, st.md_mags, (size_t)st.n_md * 4, cudaMemcpyDeviceToDevice, s));
        }
        CDB_CUDA_TRY(cudaMemcpyAsync(new_bits + (size_t)st.n_md * M, rh.md_bits, (size_t)rh.n_md * M * 4, cudaMemcpyHostToDevice, s));
        CDB_CUDA_TRY(cudaMemcpyAsync(new_mags + st.n_md, rh.md_mags, (size_t)rh.n_md * 4, cudaMemcpyHostToDevice, s));
    }
    const uint32_t *src[4] = {rh.row, rh.node_id, rh.base_id, rh.md_row};
    for (int c = 0; c < 4; ++c) CDB_CUDA_TRY(cudaMemcpyAsync(d_list + (size_t)c * n, src[c], (size_t)n * 4, cudaMemcpyHostToDevice, s));
    ReplicaDev rl = replica_table(rh.n_md ? new_bits : st.md_bits, rh.n_md ? new_mags : st.md_mags, M);
    rl.row = d_list - first;   // indexed by global list position: entry t of this call is position first + t
    rl.id = d_list + n - first;
    rl.base_id = d_list + 2 * (size_t)n - first;
    rl.md = d_list + 3 * (size_t)n - first;
    if ((rc = insert_planned(sc, gh, st, p, first, first, ef_construction, shortlist, max_batch, ~0ull, out_failed, changed, s, nullptr,
                             &rl, what)))
        return rc;
    // ---- the grown table replaces the old one
    if (rh.n_md) {
        for (const void *old : {(const void *)st.md_bits, (const void *)st.md_mags}) {
            auto it = std::find(gh.allocs->begin(), gh.allocs->end(), old);
            if (it != gh.allocs->end()) { gh.allocs->erase(it); cudaFree(const_cast<void *>(old)); }
        }
        gh.allocs->insert(gh.allocs->end(), table.p.begin(), table.p.end());
        table.release();
        st.md_bits = new_bits;
        st.md_mags = new_mags;
        st.n_md = n_md;
    }
    st.n_list += n;
    return CDB_OK;
}

// as hnsw_build_device: the two roots on every level, then the whole list through the insert path, which installs the
// Metadata table
cdb_status hnsw_build_replicas_device(const HnScoreCtx &sc, const ReplicaHost &rh, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0,
                                      uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, const GraphHost &gh,
                                      uint8_t *out_failed, const int32_t **md_bits, const float **md_mags, HnswBuildState **out_state,
                                      cudaStream_t s) {
    std::unique_ptr<HnswBuildState> st;
    cdb_status rc = new_graph(sc.metric, num_levels, nbrs, nbrs0, rh.main_root_row, 0, 0u, gh, st);
    if (rc) return rc;
    st->replicas = true;
    st->g.pseudo_entry = 1;
    st->pseudo_root_row = rh.pseudo_root_row;
    st->md_dims = rh.md_dims;
    const uint32_t L1 = num_levels + 1;
    bool changed = false;
    const std::vector<std::vector<uint32_t>> rows(L1, {rh.main_root_row, rh.pseudo_root_row}), child(L1, {0u, 1u});
    ReplicaCols cols;
    cols.id.assign(L1, {0xFFFFFFFFu, MD_PSEUDO_ID_LO});
    cols.md.assign(L1, {rh.main_root_md, rh.pseudo_root_md});
    cols.ins.assign(L1, {HN_EMPTY, HN_EMPTY});
    if ((rc = append_levels(*st, gh, rows, child, ~0ull, &changed, s, &cols)) ||
        (rc = insert_replica_list(sc, gh, *st, rh, ef_construction, shortlist, max_batch, out_failed, &changed, s, "hnsw replica build")))
        return rc;
    *md_bits = st->md_bits;
    *md_mags = st->md_mags;
    *out_state = st.release();
    return CDB_OK;
}

cdb_status hnsw_insert_replicas_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, const ReplicaHost &rh,
                                       uint32_t ef_construction, uint32_t shortlist, uint32_t max_batch, uint8_t *out_failed,
                                       const int32_t **md_bits, const float **md_mags, bool *changed, cudaStream_t s) {
    cdb_status rc = insert_replica_list(sc, gh, *st, rh, ef_construction, shortlist, max_batch, out_failed, changed, s, "hnsw replica insert");
    if (rc) return rc;
    *md_bits = st->md_bits;
    *md_mags = st->md_mags;
    return CDB_OK;
}

// ------------------------------------------------------------------ delete_embedding on a replica graph (D5)
// The unit is a vector row: every node whose node_row is the row (its base replica and its Metadata replicas, on every level)
// is deleted.  Each such node is an item: it traverses as the graph sees it (hnsw_build_search_kernel in delete mode over
// per-item arrays), then one warp per (row, level) repairs the row's nodes in list order, the sweep clears the remaining links
// to them, and the touched nodes are relinked from the candidates of the smallest item position they named.
struct DelHit { uint32_t level, node, ins, row, id, md; };

__global__ void hnsw_delete_rowset_kernel(const uint32_t *rows, uint32_t n, uint32_t *bits) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicOr(bits + (rows[i] >> 5), 1u << (rows[i] & 31));
}

// one grid-stride pass over a level's node_row: each node with a list position (not a root) whose row is in `bits` is
// counted, and with `out` set emitted (the order of the hits is the host's to fix)
__global__ void hnsw_delete_find_kernel(BuildLevel l, uint32_t level, const uint32_t *bits, uint32_t n_rows, uint32_t *n_hits,
                                        DelHit *out) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < l.cnt; j += gridDim.x * blockDim.x) {
        const uint32_t r = l.node_row[j];
        if (r >= n_rows || !bit_set(bits, r) || l.node_ins[j] == HN_EMPTY) continue;
        const uint32_t k = atomicAdd(n_hits, 1u);
        if (out) out[k] = DelHit{level, j, l.node_ins[j], r, l.node_id[j], l.node_md[j]};
    }
}

cdb_status hnsw_delete_replicas_device(const HnScoreCtx &sc, const GraphHost &gh, HnswBuildState *st, const uint32_t *rows, uint32_t n,
                                       uint32_t shortlist, uint32_t max_batch, uint8_t *out_status, bool *changed, cudaStream_t s) {
    const uint32_t L1 = st->g.num_levels + 1;
    for (uint32_t i = 0; i < n; ++i) out_status[i] = 0;
    if (!n) return CDB_OK;
    cdb_status rc;
    int sms = 0;
    if ((rc = sm_count(&sms))) return rc;
    // ---- the rows' nodes, found on the device (a replica graph has no level that lists rows in order)
    const uint32_t n_rows = *std::max_element(rows, rows + n) + 1;
    DevAllocs look;
    uint32_t *d_rows = nullptr, *d_bits = nullptr, *d_nhits = nullptr;
    DelHit *d_hits = nullptr;
    if ((rc = look.get((void **)&d_rows, (size_t)n * 4)) || (rc = look.get((void **)&d_bits, (size_t)(n_rows / 32 + 1) * 4)) ||
        (rc = look.get((void **)&d_nhits, 4)))
        return rc;
    CDB_CUDA_TRY(cudaMemcpyAsync(d_rows, rows, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    CDB_CUDA_TRY(cudaMemsetAsync(d_bits, 0, (size_t)(n_rows / 32 + 1) * 4, s));
    hnsw_delete_rowset_kernel<<<(n + 255) / 256, 256, 0, s>>>(d_rows, n, d_bits);
    CDB_LAUNCH_CHECK();
    uint32_t nh = 0;
    for (int pass = 0; pass < 2; ++pass) {   // count, then emit into an array of that size
        CDB_CUDA_TRY(cudaMemsetAsync(d_nhits, 0, 4, s));
        for (uint32_t L = 0; L < L1; ++L) {
            const BuildLevel &l = st->g.lv[L];
            if (!l.cnt) continue;
            const uint32_t grid = std::min<uint32_t>((l.cnt + 255) / 256, (uint32_t)sms * 8);
            hnsw_delete_find_kernel<<<grid, 256, 0, s>>>(l, L, d_bits, n_rows, d_nhits, d_hits);
            CDB_LAUNCH_CHECK();
        }
        CDB_CUDA_TRY(cudaMemcpyAsync(&nh, d_nhits, 4, cudaMemcpyDeviceToHost, s));
        CDB_CUDA_TRY(cudaStreamSynchronize(s));
        if (pass == 0 && !nh) return CDB_OK;   // no row of the call has a node: they are only marked
        if (pass == 0 && (rc = look.get((void **)&d_hits, (size_t)nh * sizeof(DelHit)))) return rc;
    }
    std::vector<DelHit> hits(nh);
    CDB_CUDA_TRY(cudaMemcpy(hits.data(), d_hits, (size_t)nh * sizeof(DelHit), cudaMemcpyDeviceToHost));
    // items: the level-0 nodes (every node of the list has one), by the row's position in the call, then by list position
    std::unordered_map<uint32_t, uint32_t> pos;
    for (uint32_t i = 0; i < n; ++i) pos.emplace(rows[i], i);
    std::vector<DelHit> items;
    for (const DelHit &h : hits) if (h.level == 0) items.push_back(h);
    std::sort(items.begin(), items.end(), [&](const DelHit &x, const DelHit &y) {
        const uint32_t px = pos[x.row], py = pos[y.row];
        return px != py ? px < py : x.ins < y.ins;
    });
    const uint32_t ni = (uint32_t)items.size();
    if (!ni) return CDB_OK;
    std::unordered_map<uint32_t, uint32_t> item_of;   // list position -> item
    DelItems it;
    it.loc.assign((size_t)ni * L1, HN_EMPTY);
    it.cols.resize((size_t)ni * 3);
    it.rowlist.resize(ni);
    it.out.resize(ni);
    for (uint32_t k = 0; k < ni; ++k) {
        item_of.emplace(items[k].ins, k);
        it.cols[k] = items[k].row; it.cols[ni + k] = items[k].id; it.cols[2 * (size_t)ni + k] = items[k].md;
        it.rowlist[k] = k;
        it.out[k] = pos[items[k].row];
        if (!k || it.out[k] != it.out[k - 1]) it.row_items.push_back(k);
    }
    for (const DelHit &h : hits) it.loc[(size_t)item_of.at(h.ins) * L1 + h.level] = h.node;
    it.row_items.push_back(ni);
    return delete_items(sc, st, it, shortlist, max_batch, out_status, changed, s, sms, "hnsw replica delete");
}

// ------------------------------------------------------------------ builder state of a loaded replica graph
// cdb_index_set_graph_slot_scores: the state the reference holds after a restart (ProbNode::new_with_neighbors_and_versions,
// prob_node.rs:145-181) -- every filled slot keeps the similarity stored with it on disk and lowest_index is derived afresh.
// The uploaded order stays (nothing is renumbered; searches and read_graph see the same arrays): the roots keep their local
// indices, and a loaded node's list position is the level-0 index of its node, carried up the child links (the roots have
// none).  build_local only ever searches the nodes of the current call, and the delete finds a row's nodes by a pass over
// node_row, so neither needs the loaded nodes in any order.  Inserted nodes take positions from level_counts[0] on.

// one warp per node: simkey arrives holding the stored f32 bits and becomes their order keys; a filled slot whose tag is not
// want_tag sets bit 0 of *bad
__global__ void __launch_bounds__(SS_WARPS * 32) hnsw_attach_slots_kernel(BuildLevel l, uint32_t level, const uint32_t *below_ins,
                                                                          const uint8_t *tags, uint32_t want_tag, int metric,
                                                                          uint32_t min_key, uint32_t max_key, uint32_t root0,
                                                                          uint32_t root1, uint32_t *bad) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t node = blockIdx.x * SS_WARPS + warp; node < l.cnt; node += gridDim.x * SS_WARPS) {
        SlotLowest lo;
        bool mismatch = false;
        for (uint32_t s = lane; s < l.nb; s += 32) {
            const size_t t = (size_t)node * l.nb + s;
            const bool empty = l.adj[t] == HN_EMPTY;
            const uint32_t key = empty ? 0u : order_key(metric, l.simkey[t]);
            if (!empty && tags && tags[t] != want_tag) mismatch = true;
            l.simkey[t] = key;
            lo.note(s, empty, key, max_key);
        }
        uint32_t li, lk;
        lo.finish(min_key, max_key, li, lk);
        if (mismatch) atomicOr(bad, 1u);
        if (lane == 0) {
            l.lowest_idx[node] = li;
            l.lowest_key[node] = lk;
            l.lock[node] = 0;
            const_cast<uint32_t *>(l.node_ins)[node] =
                level == 0 ? (node == root0 || node == root1 ? HN_EMPTY : node) : below_ins[l.child[node]];
        }
    }
}

// duplicate node ids on a level: open addressing over id + 1 (0 = free); an id met twice sets bit 1 of *bad
__global__ void hnsw_attach_ids_kernel(const uint32_t *ids, uint32_t cnt, unsigned long long *table, uint64_t mask, uint32_t *bad) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
        const unsigned long long v = (unsigned long long)ids[i] + 1ull;
        uint64_t h = ((uint64_t)ids[i] * 0x9E3779B97F4A7C15ull >> 24) & mask;
        for (;;) {
            const unsigned long long old = atomicCAS(table + h, 0ull, v);
            if (old == 0ull) break;
            if (old == v) { atomicOr(bad, 2u); break; }
            h = (h + 1) & mask;
        }
    }
}

// MetricResult's tag byte for the index's metric (types.rs:425-431)
static uint32_t metric_result_tag(int metric) {
    switch (metric) {
    case CDB_METRIC_COSINE: return 0;        // CosineSimilarity
    case CDB_METRIC_EUCLIDEAN: return 2;     // EuclideanDistance
    case CDB_METRIC_HAMMING: return 3;       // HammingDistance
    default: return 4;                       // DotProductDistance
    }
}

cdb_status hnsw_attach_replica_state_device(int metric, const GraphHost &gh, const float *const *scores, const uint8_t *const *tags,
                                            uint32_t pseudo_entry, uint32_t n_md, uint32_t md_dims, const int32_t *md_bits,
                                            const float *md_mags, HnswBuildState **out_state, cudaStream_t s) {
    const GraphDev &d = *gh.dev;
    const uint32_t L1 = d.num_levels + 1;
    if (L1 > BUILD_MAX_LEVELS) { set_error("the graph has more levels than the builder supports"); return CDB_UNSUPPORTED; }
    const bool has_pseudo = pseudo_entry != d.entry;
    // the roots' level-local indices, down their child links from the top level
    std::vector<uint32_t> root0(L1), root1(L1, HN_EMPTY);
    root0[L1 - 1] = d.entry;
    if (has_pseudo) root1[L1 - 1] = pseudo_entry;
    for (uint32_t L = L1 - 1; L > 0; --L) {
        CDB_CUDA_TRY(cudaMemcpy(&root0[L - 1], (*gh.ch)[L] + root0[L], 4, cudaMemcpyDeviceToHost));
        if (has_pseudo) CDB_CUDA_TRY(cudaMemcpy(&root1[L - 1], (*gh.ch)[L] + root1[L], 4, cudaMemcpyDeviceToHost));
    }
    uint32_t pseudo_row = CDB_INVALID_ID;
    if (has_pseudo) CDB_CUDA_TRY(cudaMemcpy(&pseudo_row, (*gh.nr)[L1 - 1] + pseudo_entry, 4, cudaMemcpyDeviceToHost));
    // ---- every allocation before anything changes
    std::unique_ptr<HnswBuildState> st(new HnswBuildState());
    st->g.num_levels = d.num_levels;
    st->g.entry = d.entry;
    st->g.root_row = d.root_row;
    st->g.pseudo_entry = pseudo_entry;
    metric_key_range(metric, &st->g.min_key, &st->g.max_key);
    cdb_status rc;
    DevAllocs kept, tmp;
    size_t max_slots = 0;
    uint32_t max_cnt = 0;
    for (uint32_t L = 0; L < L1; ++L) {
        BuildLevel &l = st->g.lv[L];
        l.cnt = l.app = (*gh.cnt)[L];
        l.nb = L == 0 ? d.nbrs0 : d.nbrs;
        l.node_row = const_cast<uint32_t *>((*gh.nr)[L]);
        l.adj = const_cast<uint32_t *>((*gh.ad)[L]);
        l.child = L ? const_cast<uint32_t *>((*gh.ch)[L]) : nullptr;
        l.node_id = (*gh.id)[L];
        l.node_md = (*gh.md)[L];
        st->cap[L] = l.cnt;
        const size_t slots = (size_t)l.cnt * l.nb;
        if ((rc = kept.get((void **)&l.simkey, slots * 4)) || (rc = kept.get((void **)&l.lowest_idx, (size_t)l.cnt * 4)) ||
            (rc = kept.get((void **)&l.lowest_key, (size_t)l.cnt * 4)) || (rc = kept.get((void **)&l.lock, (size_t)l.cnt * 4)) ||
            (rc = kept.get((void **)&level_array(l, 9), (size_t)l.cnt * 4)))
            return rc;
        max_slots = std::max(max_slots, slots);
        max_cnt = std::max(max_cnt, l.cnt);
    }
    uint64_t table_n = 2;
    while (table_n < 2ull * max_cnt) table_n <<= 1;
    uint8_t *d_tags = nullptr;
    unsigned long long *table = nullptr;
    uint32_t *d_bad = nullptr;
    if ((tags && (rc = tmp.get((void **)&d_tags, max_slots))) || (rc = tmp.get((void **)&table, table_n * 8)) ||
        (rc = tmp.get((void **)&d_bad, 4)))
        return rc;
    int dev = 0, sms = 0;
    CDB_CUDA_TRY(cudaGetDevice(&dev));
    CDB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    // ---- per level: the stored values in, the ids checked, keys / lowest_index / list positions derived
    CDB_CUDA_TRY(cudaMemsetAsync(d_bad, 0, 4, s));
    const uint32_t want_tag = metric_result_tag(metric);
    for (uint32_t L = 0; L < L1; ++L) {
        const BuildLevel &l = st->g.lv[L];
        const size_t slots = (size_t)l.cnt * l.nb;
        if (!l.cnt) continue;
        CDB_CUDA_TRY(cudaMemcpyAsync(l.simkey, scores[L], slots * 4, cudaMemcpyHostToDevice, s));
        if (tags) CDB_CUDA_TRY(cudaMemcpyAsync(d_tags, tags[L], slots, cudaMemcpyHostToDevice, s));
        CDB_CUDA_TRY(cudaMemsetAsync(table, 0, table_n * 8, s));
        const uint32_t id_grid = std::min<uint32_t>((l.cnt + 255) / 256, (uint32_t)sms * 8);
        hnsw_attach_ids_kernel<<<id_grid, 256, 0, s>>>(l.node_id, l.cnt, table, table_n - 1, d_bad);
        CDB_LAUNCH_CHECK();
        const uint32_t grid = std::min<uint32_t>((l.cnt + SS_WARPS - 1) / SS_WARPS, (uint32_t)sms * 16);
        hnsw_attach_slots_kernel<<<grid, SS_WARPS * 32, 0, s>>>(l, L, L ? st->g.lv[L - 1].node_ins : nullptr, tags ? d_tags : nullptr,
                                                               want_tag, metric, st->g.min_key, st->g.max_key, root0[L], root1[L], d_bad);
        CDB_LAUNCH_CHECK();
    }
    uint32_t bad = 0;
    CDB_CUDA_TRY(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error(std::string("hnsw slot scores: ") + cudaGetErrorString(e)); return CDB_CUDA_ERROR; }
    if (bad & 1u) {
        set_error("a stored slot's MetricResult tag is not the index metric's (" + std::to_string(want_tag) + ")");
        return CDB_STORAGE_MISMATCH;
    }
    if (bad & 2u) { set_error("a level of the graph lists a node id twice"); return CDB_INVALID_PARAMS; }
    // ---- the state joins the graph
    st->replicas = true;
    st->n_list = (*gh.cnt)[0];
    st->pseudo_root_row = pseudo_row;
    st->n_md = n_md;
    st->md_dims = md_dims;
    st->md_bits = md_bits;
    st->md_mags = md_mags;
    gh.allocs->insert(gh.allocs->end(), kept.p.begin(), kept.p.end());
    kept.release();
    *out_state = st.release();
    return CDB_OK;
}

}  // namespace cdb
