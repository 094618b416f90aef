/*
 * hnsw_loaded_md_oracle.c -- TEST INFRASTRUCTURE ONLY: the replica oracle's builder state reloaded from level arrays and the
 * similarities stored with their slots, as a restart of the reference holds it (ProbNode::new_with_neighbors_and_versions,
 * prob_node.rs:145-181): every filled slot keeps its stored value, lowest_index is derived afresh -- the first empty slot
 * gives MetricResult::min, otherwise, scanning from MetricResult::max, the first slot with a strictly lower key.  It
 * #includes the delete oracle so that mdo_insert / mdo_delete_rows continue on the reloaded state.
 * List positions follow cdb_index_set_graph_slot_scores: a loaded node's position is the level-0 index of its node (carried
 * up the child links), the roots have none, and entries inserted later follow from level_counts[0] on.  The delete oracle
 * finds a row's nodes behind local index 1, so mdo_load takes every level with the main root at local 0 and the pseudo root
 * at local 1 and refuses other layouts; pos0 (may be NULL = the level-0 index) gives each level-0 node's list position, so a
 * caller may renumber a graph into that layout and keep the positions it had.  A graph without a pseudo root (a collection
 * without a metadata schema) is loaded with an isolated placeholder at local 1 that no traversal reaches: its inserts must
 * not carry pseudo replicas or Metadata with mag != 0 (tests/scored_index_files.py refuses them).
 */
#include "hnsw_delete_md_oracle.c"

/* lowest_index of one node from its slots (adj / simkey, nb of them) */
void mdo_lowest(const uint32_t *adj, const uint32_t *simkey, uint32_t nb, uint32_t min_key, uint32_t max_key, uint32_t *li,
                uint32_t *lk) {
    *li = 0;
    *lk = max_key;
    for (uint32_t s = 0; s < nb; ++s) {
        if (adj[s] == ORC_EMPTY) { *li = s; *lk = min_key; return; }
        if (simkey[s] < *lk) { *li = s; *lk = simkey[s]; }
    }
}

void mdo_key_range(int metric, uint32_t *min_key, uint32_t *max_key) { bl_min_max_keys(metric, min_key, max_key); }

/* counts[L], node_row / node_id / node_md / child [L][counts[L]], adj / scores [L][counts[L] * nbrs(L)] (level 0: nbrs0);
 * entry / pseudo_entry: top-level indices (0 and 1).  NULL when the roots are not local 0 / 1 on every level. */
mdo *mdo_load(int metric, int st, size_t dim, const void *codes, const float *mags, size_t md_dims, const int32_t *md_bits,
              const float *md_mags, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0, const uint32_t *counts,
              const uint32_t *const *node_row, const uint32_t *const *node_id, const uint32_t *const *node_md,
              const uint32_t *const *adj, const uint32_t *const *child, const float *const *scores, const uint32_t *pos0) {
    const uint32_t L1 = num_levels + 1, top = num_levels;
    if (L1 > 16 || counts[top] < 2) return NULL;
    for (uint32_t L = top; L > 0; --L)
        if (child[L][0] != 0 || child[L][1] != 1) return NULL;
    mdo *o = mdo_new(metric, st, dim, codes, mags, md_dims, md_bits, md_mags, num_levels, nbrs, nbrs0, node_row[top][0],
                     node_md[top][0], node_row[top][1], node_md[top][1]);
    if (!o) return NULL;
    orc_md_built *b = o->b;
    for (uint32_t L = 0; L < L1; ++L) {
        blevel *l = &b->lv[L];
        const uint32_t cnt = counts[L], nb = l->nb;
        lv_reserve(l, cnt);
        ins_reserve(o, L);
        l->cnt = cnt;
        for (uint32_t i = 0; i < cnt; ++i) {
            l->node_row[i] = node_row[L][i];
            l->node_id[i] = node_id[L][i];
            l->node_md[i] = node_md[L][i];
            l->child[i] = L ? child[L][i] : ORC_EMPTY;
            for (uint32_t s = 0; s < nb; ++s) {
                const size_t t = (size_t)i * nb + s;
                l->adj[t] = adj[L][t];
                l->simkey[t] = adj[L][t] == ORC_EMPTY ? 0u : orc_order_key(metric, scores[L][t]);
            }
            mdo_lowest(l->adj + (size_t)i * nb, l->simkey + (size_t)i * nb, nb, b->min_key, b->max_key, &l->lowest_idx[i],
                       &l->lowest_key[i]);
            o->ins[L][i] = i < 2 ? ORC_EMPTY : (L ? o->ins[L - 1][child[L][i]] : (pos0 ? pos0[i] : i));
        }
    }
    /* the list: position ins[0][i] = level-0 node i (positions without a node hold no entry) */
    uint32_t n0 = 0;
    for (uint32_t i = 2; i < counts[0]; ++i)
        if (o->ins[0][i] + 1 > n0) n0 = o->ins[0][i] + 1;
    o->list_cap = n0 ? n0 : 1;
    o->row = (uint32_t *)malloc(sizeof(uint32_t) * o->list_cap);
    o->node_id = (uint32_t *)malloc(sizeof(uint32_t) * o->list_cap);
    o->base_id = (uint32_t *)malloc(sizeof(uint32_t) * o->list_cap);
    o->md_row = (uint32_t *)malloc(sizeof(uint32_t) * o->list_cap);
    for (uint32_t t = 0; t < n0; ++t) o->row[t] = o->node_id[t] = o->base_id[t] = o->md_row[t] = ORC_EMPTY;
    for (uint32_t i = 2; i < counts[0]; ++i) {
        const uint32_t t = o->ins[0][i];
        o->row[t] = node_row[0][i];
        o->node_id[t] = o->base_id[t] = node_id[0][i];
        o->md_row[t] = node_md[0][i];
    }
    o->n_list = n0;
    md_refresh_view(b);
    return o;
}
