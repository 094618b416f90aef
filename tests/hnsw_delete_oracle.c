/*
 * hnsw_delete_oracle.c -- TEST INFRASTRUCTURE ONLY: deterministic single-threaded restatement of delete_embedding
 * (src/vector_store.rs:1206-1371) on the insert oracle's live graph, with the deviations of cdb_index_delete_rows:
 *   D1 the deleted node D is unlinked on every level it is on, whether or not the ef-512 traversal found it;
 *   D2 after D's own slots, every remaining slot naming D is cleared, then each node that lost a slot that way is relinked,
 *      in ascending level-local index, if its list is empty at its turn;
 *   D3 an Err stops relinks (a traversal Err: that level and below; a rescoring Err: that one relink), not unlinking;
 *   D4 D keeps its nodes, isolated (lowest_index reset to (0, MetricResult::min)).
 * Rows are deleted one at a time in list order, which is what the GPU does with max_batch = 1.
 */
#include "hnsw_insert_oracle.c"

#define DEL_EF 512u    /* the reference's literal ef (vector_store.rs:1247) */
#define DEL_KEEP 100u  /* final_len when not indexing (vector_store.rs:1194) */

static int del_remove_by_id(blevel *l, uint32_t node, uint32_t id) { /* remove_neighbor_by_id: lowest_index stays stale */
    for (uint32_t s = 0; s < l->nb; ++s)
        if (l->adj[(size_t)node * l->nb + s] == id) { l->adj[(size_t)node * l->nb + s] = ORC_EMPTY; return 1; }
    return 0;
}
static int del_is_empty(const blevel *l, uint32_t node) {
    for (uint32_t s = 0; s < l->nb; ++s)
        if (l->adj[(size_t)node * l->nb + s] != ORC_EMPTY) return 0;
    return 1;
}

/* the relink of an emptied node N (vector_store.rs:1306-1357): the results minus D, N and deleted rows, rescored against N
 * (calculate(N, entry)), sorted best first (ties: smaller id), through create_node_edges.  Returns the rescoring's rc. */
static int del_relink(ig *g, blevel *l, uint32_t N, uint32_t D, const uint32_t *res, uint32_t nres, const uint8_t *deleted) {
    hitem cand[DEL_KEEP];
    uint32_t m = 0, nodes[DEL_KEEP];
    float scores[DEL_KEEP];
    const uint32_t nrow = l->node_row[N];
    for (uint32_t i = 0; i < nres; ++i) {
        const uint32_t c = res[i], crow = l->node_row[c];
        if (c == D || c == N || deleted[crow]) continue;
        float d;
        int rc = orc_distance(g->metric, g->st, g->dim, ig_code(g, nrow), g->mags[nrow], ig_code(g, crow), g->mags[crow], &d);
        if (rc != ORC_OK) return rc;
        cand[m++] = (hitem){ig_key(g, d, ig_id(g, crow)), c, d};
    }
    qsort(cand, m, sizeof(hitem), cmp_desc);
    for (uint32_t i = 0; i < m; ++i) { nodes[i] = cand[i].node; scores[i] = cand[i].score; }
    create_node_edges(g, l, N, nodes, scores, m);
    return ORC_OK;
}

/* deletes rows[0..n) one at a time.  deleted[table rows] is the caller's deletion mask (read and updated).
 * out_status[i]: 0 deleted, 1 already deleted, 2 deleted but an Err stopped relinks. */
void ig_delete_rows(ig *g, const uint32_t *rows, uint32_t n, uint32_t shortlist, uint8_t *deleted, uint8_t *out_status) {
    uint32_t maxnb = 0, maxcnt = 0;
    for (uint32_t L = 0; L <= g->num_levels; ++L) {
        if (g->lv[L].nb > maxnb) maxnb = g->lv[L].nb;
        if (g->lv[L].cnt > maxcnt) maxcnt = g->lv[L].cnt;
    }
    uint64_t *fs = (uint64_t *)malloc(sizeof(uint64_t) * maxnb);
    uint8_t *touched = (uint8_t *)malloc(maxcnt ? maxcnt : 1);
    uint32_t res[DEL_KEEP];
    float rs[DEL_KEEP];
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t r = rows[i];
        if (deleted[r]) { out_status[i] = 1; continue; }
        deleted[r] = 1;
        out_status[i] = 0;
        if (r >= g->lv[0].cnt) continue;   /* not in the graph: only marked */
        uint32_t entry = g->entry;
        int err = 0;
        for (int level = (int)g->num_levels; level >= 0; --level) {
            blevel *l = &g->lv[level];
            uint32_t nres = 0;
            if (!err) {   /* a fresh fixed set, nothing pre-inserted (vector_store.rs:1231-1235) */
                memset(fs, 0, sizeof(uint64_t) * l->nb);
                if (ig_traverse(g, (uint32_t)level, entry, ig_code(g, r), g->mags[r], DEL_EF, shortlist, DEL_KEEP, fs, res, rs, &nres,
                                NULL, NULL) != ORC_OK) {
                    err = 1;   /* D3: no relinks on this level or below */
                    out_status[i] = 2;
                } else if (level > 0) {
                    entry = l->child[res[0]];
                }
            }
            uint32_t D = ORC_EMPTY;   /* D1: D's node on this level, found or not */
            if (level == 0) D = r;
            else for (uint32_t j = 0; j < l->cnt && D == ORC_EMPTY; ++j) if (l->node_row[j] == r) D = j;
            if (D == ORC_EMPTY) continue;
            for (uint32_t s = 0; s < l->nb; ++s) {
                const uint32_t N = l->adj[(size_t)D * l->nb + s];
                if (N == ORC_EMPTY) continue;
                if (del_remove_by_id(l, N, D) && !deleted[l->node_row[N]] && del_is_empty(l, N) && !err &&
                    del_relink(g, l, N, D, res, nres, deleted) != ORC_OK)
                    out_status[i] = 2;
            }
            for (uint32_t s = 0; s < l->nb; ++s) l->adj[(size_t)D * l->nb + s] = ORC_EMPTY;   /* D4 */
            l->lowest_idx[D] = 0;
            l->lowest_key[D] = g->min_key;
            /* D2: the links to D from outside its list */
            memset(touched, 0, l->cnt);
            for (uint32_t x = 0; x < l->cnt; ++x)
                for (uint32_t s = 0; s < l->nb; ++s)
                    if (l->adj[(size_t)x * l->nb + s] == D) { l->adj[(size_t)x * l->nb + s] = ORC_EMPTY; touched[x] = 1; }
            for (uint32_t x = 0; x < l->cnt; ++x)
                if (touched[x] && !deleted[l->node_row[x]] && del_is_empty(l, x) && !err &&
                    del_relink(g, l, x, D, res, nres, deleted) != ORC_OK)
                    out_status[i] = 2;
        }
    }
    free(fs);
    free(touched);
}
