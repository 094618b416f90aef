/*
 * hnsw_insert_oracle.c -- TEST INFRASTRUCTURE ONLY: deterministic single-threaded restatement of index_embeddings on a
 * LIVE graph (src/vector_store.rs:714-940), the CPU side of cdb_index_insert_graph.
 *
 * Unlike oracle/hnsw_oracle.c, whose flat graph has the root as the last row, the root here is any row (`root_row`):
 * after an insert the root sits between the rows of the first build and the rows inserted later.  The builder is split
 * into ig_init (the root on every level) + ig_insert_rows, and tests pin ig_init + ig_insert_rows(0, n) to
 * orc_hnsw_build(n) array for array, so the insert path is the builder the existing oracle tests pin.
 *   ig_from_graph   a graph loaded from storage: sims recomputed, lowest_index per ProbNode::new_with_neighbors_and_versions
 *                   (src/models/prob_node.rs:145-181)
 *   ig_search_batch search_internal on the graph (src/indexes/hnsw/mod.rs:390-440), ids = rows, root = u32::MAX
 * Level layout: level 0 node i = row i; levels >= 1: the root, then each call's rows ascending (nodes of all levels a
 * row reaches are created before its traversal, so a failed insert leaves them unlinked).
 */
#include <stdlib.h>
#include <string.h>

#include "hnsw_build_internal.h"

typedef struct {
    int metric, st;
    size_t dim, cb;
    const uint8_t *codes;   /* the caller's table, >= every row the graph names */
    const float *mags;
    uint32_t num_levels, entry, root_row, min_key, max_key;
    blevel *lv;
    uint32_t *app;          /* first node appended by the current insert, per level */
} ig;

static inline uint32_t ig_id(const ig *g, uint32_t row) { return row == g->root_row ? ORC_ROOT_ID : row; }
static inline const uint8_t *ig_code(const ig *g, uint32_t row) { return g->codes + (size_t)row * g->cb; }
static inline uint64_t ig_key(const ig *g, float score, uint32_t id) {
    return ((uint64_t)orc_order_key(g->metric, score) << 32) | (uint64_t)(~id);
}
static inline void fs_insert(uint64_t *b, uint32_t len, uint32_t v) { b[(v >> 6) & (len - 1u)] |= 1ull << (v & 0x3f); }
static inline int fs_member(const uint64_t *b, uint32_t len, uint32_t v) { return (b[(v >> 6) & (len - 1u)] >> (v & 0x3f)) & 1ull; }

typedef struct { uint64_t key; uint32_t node; float score; } hitem;
static void heap_push(hitem *h, size_t *n, hitem it) {
    size_t i = (*n)++;
    h[i] = it;
    while (i > 0) {
        size_t p = (i - 1) / 2;
        if (h[p].key >= h[i].key) break;
        hitem t = h[p]; h[p] = h[i]; h[i] = t;
        i = p;
    }
}
static hitem heap_pop(hitem *h, size_t *n) {
    hitem top = h[0];
    h[0] = h[--(*n)];
    size_t i = 0;
    for (;;) {
        size_t l = 2 * i + 1, r = l + 1, m = i;
        if (l < *n && h[l].key > h[m].key) m = l;
        if (r < *n && h[r].key > h[m].key) m = r;
        if (m == i) break;
        hitem t = h[m]; h[m] = h[i]; h[i] = t;
        i = m;
    }
    return top;
}
static int cmp_desc(const void *a, const void *b) {
    uint64_t x = ((const hitem *)a)->key, y = ((const hitem *)b)->key;
    return (x < y) - (x > y);
}

/* traverse_find_nearest (src/vector_store.rs:1112-1204) on one level */
static int ig_traverse(const ig *g, uint32_t level, uint32_t entry, const uint8_t *q, float qmag, uint32_t ef, uint32_t shortlist,
                       uint32_t final_len, uint64_t *fs, uint32_t *out_nodes, float *out_scores, uint32_t *out_n, uint64_t *evals,
                       uint64_t *pops) {
    const blevel *l = &g->lv[level];
    const uint32_t nb = l->nb, take = shortlist < nb ? shortlist : nb;
    size_t hn = 0, rn = 0;
    hitem *heap = (hitem *)malloc(sizeof(hitem) * ((size_t)ef * take + 2));
    hitem *res = (hitem *)malloc(sizeof(hitem) * ((size_t)ef + 1));
    float d;
    uint32_t erow = l->node_row[entry];
    int rc = orc_distance(g->metric, g->st, g->dim, q, qmag, ig_code(g, erow), g->mags[erow], &d);
    if (evals) (*evals)++;
    if (rc != ORC_OK) goto done;
    fs_insert(fs, nb, ig_id(g, erow));
    heap_push(heap, &hn, (hitem){ig_key(g, d, ig_id(g, erow)), entry, d});
    uint32_t visited = 0;
    while (hn > 0) {
        hitem cur = heap_pop(heap, &hn);
        if (visited >= ef) break;
        visited++;
        if (pops) (*pops)++;
        res[rn++] = cur;
        const uint32_t *slots = l->adj + (size_t)cur.node * nb;
        for (uint32_t s = 0; s < take; ++s) {
            uint32_t nbl = slots[s];
            if (nbl == ORC_EMPTY) continue;
            uint32_t nrow = l->node_row[nbl], nid = ig_id(g, nrow);
            if (fs_member(fs, nb, nid)) continue;
            rc = orc_distance(g->metric, g->st, g->dim, q, qmag, ig_code(g, nrow), g->mags[nrow], &d);
            if (evals) (*evals)++;
            if (rc != ORC_OK) goto done;
            fs_insert(fs, nb, nid);
            heap_push(heap, &hn, (hitem){ig_key(g, d, nid), nbl, d});
        }
    }
    qsort(res, rn, sizeof(hitem), cmp_desc);
    if (rn > final_len) rn = final_len;
    for (size_t i = 0; i < rn; ++i) { out_nodes[i] = res[i].node; out_scores[i] = res[i].score; }
    *out_n = (uint32_t)rn;
done:
    free(heap);
    free(res);
    return rc;
}

static ig *ig_alloc(int metric, int st, size_t dim, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0) {
    ig *g = (ig *)calloc(1, sizeof(ig));
    g->metric = metric; g->st = st; g->dim = dim; g->cb = orc_code_bytes(st, dim);
    g->num_levels = num_levels;
    bl_min_max_keys(metric, &g->min_key, &g->max_key);
    g->lv = (blevel *)calloc(num_levels + 1, sizeof(blevel));
    g->app = (uint32_t *)calloc(num_levels + 1, sizeof(uint32_t));
    for (uint32_t L = 0; L <= num_levels; ++L) g->lv[L].nb = L == 0 ? nbrs0 : nbrs;
    return g;
}

/* the root on every level (vector_store.rs:44-140); level 0 holds a (not yet linked) node for each of rows 0..n_level0-1 */
ig *ig_init(int metric, int st, size_t dim, uint32_t root_row, uint32_t n_level0, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0) {
    ig *g = ig_alloc(metric, st, dim, num_levels, nbrs, nbrs0);
    g->root_row = root_row;
    for (uint32_t L = 0; L <= num_levels; ++L) {
        blevel *l = &g->lv[L];
        if (L == 0) { lv_reserve(l, n_level0); for (uint32_t i = 0; i < n_level0; ++i) lv_init_node(g->min_key, l, i, i); l->cnt = n_level0; }
        else { lv_reserve(l, 1); lv_init_node(g->min_key, l, 0, root_row); l->child[0] = L == 1 ? root_row : 0; l->cnt = 1; }
    }
    g->entry = num_levels == 0 ? root_row : 0;
    return g;
}

void ig_set_table(ig *g, const void *codes, const float *mags) { g->codes = (const uint8_t *)codes; g->mags = mags; }

static float rng_unit(uint64_t seed, uint64_t i) { /* the builders' stand-in for rand::random::<f32>() */
    uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z = z ^ (z >> 31);
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}
static uint32_t seeded_level(uint64_t seed, uint32_t row, uint32_t num_levels) { /* get_max_insert_level, probs 1 - 4^-n */
    double x = (double)rng_unit(seed, row);
    for (int lv = (int)num_levels; lv >= 0; --lv) {
        double p4 = 1.0;
        for (int e = 0; e < lv; ++e) p4 *= 4.0;
        if (x >= 1.0 - 1.0 / p4) return (uint32_t)lv;
    }
    return 0;
}

static uint32_t local_of(const ig *g, uint32_t level, uint32_t row) {
    if (level == 0) return row;
    const blevel *l = &g->lv[level];
    for (uint32_t i = g->app[level]; i < l->cnt; ++i)
        if (l->node_row[i] == row) return i;
    return ORC_EMPTY;
}

/* create_node_edges (src/vector_store.rs:976-1070), Base nodes only */
static void create_node_edges(ig *g, blevel *l, uint32_t node, const uint32_t *zn_nodes, const float *zs, uint32_t zn) {
    uint32_t successful = 0;
    for (uint32_t i = 0; i < zn; ++i) {
        if (successful >= l->nb) break;
        uint32_t nbr = zn_nodes[i], dkey = orc_order_key(g->metric, zs[i]);
        int idx = bl_add_neighbor(g->min_key, g->max_key, l, node, nbr, dkey);
        if (idx >= 0) {
            int j = bl_add_neighbor(g->min_key, g->max_key, l, nbr, node, dkey);
            if (j >= 0) successful++;
            else if (l->adj[(size_t)node * l->nb + idx] == nbr) l->adj[(size_t)node * l->nb + idx] = ORC_EMPTY;
        }
    }
}

/* index_embeddings for rows [first, first+count) in ascending order.  levels: the caller's draws (clamped) or NULL for the
 * seeded draws.  failed[count] (may be NULL): 1 where the reference's insert returns Err. */
void ig_insert_rows(ig *g, uint32_t first, uint32_t count, const uint8_t *levels, uint64_t seed, uint32_t ef, uint32_t shortlist,
                    uint8_t *failed) {
    const uint32_t L1 = g->num_levels + 1;
    uint32_t *lvl = (uint32_t *)malloc(sizeof(uint32_t) * (count ? count : 1));
    for (uint32_t i = 0; i < count; ++i) {
        uint32_t m = levels ? levels[i] : seeded_level(seed, first + i, g->num_levels);
        lvl[i] = m < g->num_levels ? m : g->num_levels;
    }
    /* nodes up front: level 0 grows to cover the rows, levels >= 1 append their rows ascending */
    for (uint32_t L = 0; L < L1; ++L) g->app[L] = g->lv[L].cnt;
    blevel *l0 = &g->lv[0];
    if (first + count > l0->cnt) {
        lv_reserve(l0, first + count);
        for (uint32_t r = l0->cnt; r < first + count; ++r) lv_init_node(g->min_key, l0, r, r);
        l0->cnt = first + count;
    }
    for (uint32_t L = 1; L < L1; ++L) {
        blevel *l = &g->lv[L];
        uint32_t j = g->app[L - 1];
        for (uint32_t i = 0; i < count; ++i) {
            if (lvl[i] < L) continue;
            uint32_t r = first + i;
            lv_reserve(l, l->cnt + 1);
            lv_init_node(g->min_key, l, l->cnt, r);
            if (L == 1) l->child[l->cnt] = r;
            else { while (g->lv[L - 1].node_row[j] != r) ++j; l->child[l->cnt] = j; }
            l->cnt++;
        }
    }
    uint32_t maxnb = 0;
    for (uint32_t L = 0; L < L1; ++L) if (g->lv[L].nb > maxnb) maxnb = g->lv[L].nb;
    uint64_t *fs = (uint64_t *)malloc(sizeof(uint64_t) * maxnb);
    uint32_t *znodes = (uint32_t *)malloc(sizeof(uint32_t) * 64 * L1);
    float *zscores = (float *)malloc(sizeof(float) * 64 * L1);
    uint32_t *zn = (uint32_t *)malloc(sizeof(uint32_t) * L1);
    for (uint32_t i = 0; i < count; ++i) {
        const uint32_t r = first + i;
        const uint8_t *code = ig_code(g, r);
        uint32_t entry = g->entry;
        int bad = 0;
        for (int level = (int)g->num_levels; level >= 0; --level) {
            blevel *l = &g->lv[level];
            memset(fs, 0, sizeof(uint64_t) * l->nb);
            fs_insert(fs, l->nb, r);
            uint32_t *zl = znodes + 64 * level;
            float *sl = zscores + 64 * level;
            uint32_t cnt = 0;
            int rc = ig_traverse(g, (uint32_t)level, entry, code, g->mags[r], ef, shortlist, 64, fs, zl, sl, &cnt, NULL, NULL);
            if (rc != ORC_OK) { bad = 1; break; }
            zn[level] = cnt;
            if (level > 0) entry = l->child[zl[0]];
        }
        if (failed) failed[i] = (uint8_t)bad;
        if (bad) continue;
        for (uint32_t level = 0; level <= lvl[i]; ++level)
            create_node_edges(g, &g->lv[level], local_of(g, level, r), znodes + 64 * level, zscores + 64 * level, zn[level]);
    }
    free(lvl); free(fs); free(znodes); free(zscores); free(zn);
}

/* a graph loaded from storage (cdb_index_set_graph): ProbNode::new_with_neighbors_and_versions (prob_node.rs:145-181) */
ig *ig_from_graph(int metric, int st, size_t dim, const void *codes, const float *mags, uint32_t root_row, uint32_t entry,
                  uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0, const uint32_t *cnt, const uint32_t *const *node_row,
                  const uint32_t *const *adj, const uint32_t *const *child) {
    ig *g = ig_alloc(metric, st, dim, num_levels, nbrs, nbrs0);
    ig_set_table(g, codes, mags);
    g->root_row = root_row;
    g->entry = entry;
    for (uint32_t L = 0; L <= num_levels; ++L) {
        blevel *l = &g->lv[L];
        lv_reserve(l, cnt[L] ? cnt[L] : 1);
        l->cnt = cnt[L];
        for (uint32_t i = 0; i < l->cnt; ++i) {
            lv_init_node(g->min_key, l, i, node_row[L][i]);
            l->child[i] = L ? child[L][i] : ORC_EMPTY;
            uint32_t nidx = 0, nkey = g->max_key, found_empty = 0;
            for (uint32_t s = 0; s < l->nb; ++s) {
                uint32_t nbl = adj[L][(size_t)i * l->nb + s], key = 0;
                l->adj[(size_t)i * l->nb + s] = nbl;
                if (nbl != ORC_EMPTY) {
                    uint32_t x = node_row[L][i], y = node_row[L][nbl];
                    float d;
                    int rc = orc_distance(metric, st, dim, ig_code(g, x), mags[x], ig_code(g, y), mags[y], &d);
                    key = rc == ORC_OK ? orc_order_key(metric, d) : g->min_key;   /* an Err pair: evicted first */
                }
                l->simkey[(size_t)i * l->nb + s] = key;
                if (found_empty) continue;
                if (nbl == ORC_EMPTY) { nidx = s; nkey = g->min_key; found_empty = 1; }
                else if (key < nkey) { nidx = s; nkey = key; }
            }
            l->lowest_idx[i] = nidx;
            l->lowest_key[i] = nkey;
        }
    }
    return g;
}

uint32_t ig_level_count(const ig *g, uint32_t level) { return g->lv[level].cnt; }
uint32_t ig_entry(const ig *g) { return g->entry; }
/* any output may be NULL; simkey is the order key of each slot (0 where never filled) */
void ig_level_export(const ig *g, uint32_t level, uint32_t *node_row, uint32_t *adj, uint32_t *child, uint32_t *simkey,
                     uint32_t *lowest_idx, uint32_t *lowest_key) {
    const blevel *l = &g->lv[level];
    const size_t c = l->cnt, s = c * l->nb;
    if (node_row) memcpy(node_row, l->node_row, c * 4);
    if (adj) memcpy(adj, l->adj, s * 4);
    if (child) memcpy(child, l->child, c * 4);
    if (simkey) memcpy(simkey, l->simkey, s * 4);
    if (lowest_idx) memcpy(lowest_idx, l->lowest_idx, c * 4);
    if (lowest_key) memcpy(lowest_key, l->lowest_key, c * 4);
}

/* search_internal for a batch (quantized ann_search, remove_duplicates_and_filter, exact f32 re-rank), one thread */
void ig_search_batch(const ig *g, const float *raw, const float *queries, size_t nq, float lo, float hi, uint32_t ef,
                     uint32_t shortlist, size_t k, uint32_t *out_ids, float *out_scores, uint32_t *out_counts, uint8_t *err,
                     uint64_t *evals, uint64_t *pops) {
    const size_t cap = ((size_t)g->num_levels + 1) * 100;
    uint32_t maxnb = 0;
    for (uint32_t L = 0; L <= g->num_levels; ++L) if (g->lv[L].nb > maxnb) maxnb = g->lv[L].nb;
    uint64_t *fs = (uint64_t *)malloc(sizeof(uint64_t) * maxnb);
    uint8_t *qcode = (uint8_t *)malloc(g->cb ? g->cb : 1);
    uint32_t *rows = (uint32_t *)malloc(sizeof(uint32_t) * cap), nodes[128];
    float *sc = (float *)malloc(sizeof(float) * cap), scores[128];
    hitem *tmp = (hitem *)malloc(sizeof(hitem) * cap);
    for (size_t qi = 0; qi < nq; ++qi) {
        const float *q = queries + qi * g->dim;
        float qmag;
        orc_quantize(g->st, lo, hi, q, g->dim, qcode, &qmag);
        size_t total = 0;
        uint32_t entry = g->entry;
        int rc = ORC_OK;
        for (int level = (int)g->num_levels; level >= 0; --level) {
            const blevel *l = &g->lv[level];
            uint32_t zn = 0;
            memset(fs, 0, sizeof(uint64_t) * l->nb);
            fs_insert(fs, l->nb, ORC_QUERY_ID);
            rc = ig_traverse(g, (uint32_t)level, entry, qcode, qmag, ef, shortlist, 100, fs, nodes, scores, &zn, evals, pops);
            if (rc != ORC_OK) break;
            for (uint32_t i = 0; i < zn && total < cap; ++i) { rows[total] = l->node_row[nodes[i]]; sc[total] = scores[i]; total++; }
            if (level > 0) entry = l->child[nodes[0]];
        }
        for (size_t j = 0; j < k; ++j) { out_ids[qi * k + j] = 0xFFFFFFFFu; out_scores[qi * k + j] = 0.0f; }
        if (rc != ORC_OK) { err[qi] = (uint8_t)(rc == ORC_CALCULATION_ERROR ? 1 : 2); out_counts[qi] = 0; continue; }
        err[qi] = 0;
        size_t m = 0;
        for (size_t i = 0; i < total; ++i) {
            int seen = 0;
            for (size_t j = 0; j < i && !seen; ++j) seen = rows[j] == rows[i];
            if (seen || ig_id(g, rows[i]) == ORC_ROOT_ID) continue;
            tmp[m++] = (hitem){ig_key(g, sc[i], rows[i]), rows[i], sc[i]};
        }
        qsort(tmp, m, sizeof(hitem), cmp_desc);
        if (m > 5 * k) m = 5 * k;
        for (size_t i = 0; i < m; ++i) rows[i] = tmp[i].node;
        orc_rerank_f32(raw, g->dim, q, rows, m, k, out_ids + qi * k, out_scores + qi * k);
        out_counts[qi] = (uint32_t)(m < k ? m : k);
    }
    free(fs); free(qcode); free(rows); free(sc); free(tmp);
}

void ig_free(ig *g) {
    if (!g) return;
    for (uint32_t L = 0; L <= g->num_levels; ++L) lv_free(&g->lv[L]);
    free(g->lv); free(g->app); free(g);
}
