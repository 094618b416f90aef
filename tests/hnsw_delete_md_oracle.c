/*
 * hnsw_delete_md_oracle.c -- TEST INFRASTRUCTURE ONLY: deterministic single-threaded restatement of delete_embedding on a
 * graph with replica nodes (a collection with a metadata schema), with the deviations of cdb_index_delete_rows_replicas.
 * It #includes the replica oracle's source so it works on that builder's own state (orc_md_built: slot similarities, stale
 * lowest_index, node ids and Metadata rows), and keeps beside it what the delete needs:
 *   - the list of entries inserted so far (row, node_id, base_id, md_row per list position), and
 *   - per level, the list position of every node (the roots: ORC_EMPTY).
 * mdo_insert continues the replica build on that state: its per-entry body is orc_hnsw_build_md's loop body restated (the
 * CPU tests pin the two against each other), plus the list positions.
 * The delete (rows one at a time, in list order -- what the GPU does with max_batch = 1):
 *   the unit is a vector row: its items are the list entries with that row, in list order.  Every item traverses the graph as
 *   of the row's start from the pseudo root (metadata with mag != 0) or the main root, carrying its row's code, its Metadata
 *   row and Some(node_id), nothing pre-inserted, ef 512, best 100 kept (a traversal Err: no relinks on that level and below);
 *   then per level the items' nodes repair their own slots in list order (D1, D3, D4); then the D2 sweep clears every slot
 *   naming a node of the row and relinks each node it touched, in ascending level-local index, from the candidates of the
 *   first item (in list order) whose node it named.  A relink rescores the candidates with the replica arms
 *   (calculate(N, candidate)), sorts them best first (ties: smaller id) and runs create_node_edges with the replica rules.
 */
#include "metadata_oracle.c"

#define DEL_EF 512u    /* the reference's literal ef (vector_store.rs:1247) */
#define DEL_KEEP 100u  /* final_len when not indexing (vector_store.rs:1194) */

typedef struct {
    orc_md_built *b;
    uint32_t *ins[16], ins_cap[16];
    uint32_t n_list, list_cap;
    uint32_t *row, *node_id, *base_id, *md_row;
} mdo;

static void ins_reserve(mdo *o, uint32_t L) {
    if (o->ins_cap[L] >= o->b->lv[L].cap) return;
    o->ins[L] = (uint32_t *)realloc(o->ins[L], sizeof(uint32_t) * o->b->lv[L].cap);
    o->ins_cap[L] = o->b->lv[L].cap;
}

/* the two roots on every level, as orc_hnsw_build_md creates them (an empty list) */
mdo *mdo_new(int metric, int st, size_t dim, const void *codes, const float *mags, size_t md_dims, const int32_t *md_bits,
             const float *md_mags, uint32_t num_levels, uint32_t nbrs, uint32_t nbrs0, uint32_t main_root_row, uint32_t main_root_md,
             uint32_t pseudo_root_row, uint32_t pseudo_root_md) {
    if (num_levels + 1 > 16) return NULL;
    orc_replica_list rl;
    memset(&rl, 0, sizeof rl);
    rl.main_root_row = main_root_row; rl.main_root_md = main_root_md;
    rl.pseudo_root_row = pseudo_root_row; rl.pseudo_root_md = pseudo_root_md;
    mdo *o = (mdo *)calloc(1, sizeof(mdo));
    o->b = orc_hnsw_build_md(metric, st, dim, codes, mags, md_dims, md_bits, md_mags, &rl, num_levels, nbrs, nbrs0, 1, 1, NULL);
    for (uint32_t L = 0; L <= num_levels; ++L) {
        ins_reserve(o, L);
        o->ins[L][0] = o->ins[L][1] = ORC_EMPTY;
    }
    return o;
}

void mdo_free(mdo *o) {
    if (!o) return;
    for (int L = 0; L < 16; ++L) free(o->ins[L]);
    free(o->row); free(o->node_id); free(o->base_id); free(o->md_row);
    orc_md_built_free(o->b);
    free(o);
}

/* index_embeddings over more list entries (orc_hnsw_build_md's loop body, continued on the same state) */
void mdo_insert(mdo *o, const orc_replica_list *rl, uint32_t ef_construction, uint32_t shortlist, uint8_t *failed_out) {
    orc_md_built *b = o->b;
    orc_md_graph *mg = &b->mg;
    orc_graph *g = &mg->g;
    const uint32_t num_levels = g->num_levels, L1 = num_levels + 1;
    const uint32_t maxnb = g->level0_neighbors_count > g->neighbors_count ? g->level0_neighbors_count : g->neighbors_count;
    uint64_t *fs = (uint64_t *)malloc(sizeof(uint64_t) * maxnb);
    mitem *z = (mitem *)malloc(sizeof(mitem) * 64 * L1);
    uint32_t *zn = (uint32_t *)malloc(sizeof(uint32_t) * L1);
    uint32_t *node_at = (uint32_t *)malloc(sizeof(uint32_t) * L1);
    const size_t cb = orc_code_bytes(g->storage_type, g->dim);
    if (o->n_list + rl->n_nodes > o->list_cap) {
        o->list_cap = (o->n_list + rl->n_nodes) * 2;
        uint32_t **cols[4] = {&o->row, &o->node_id, &o->base_id, &o->md_row};
        for (int c = 0; c < 4; ++c) *cols[c] = (uint32_t *)realloc(*cols[c], sizeof(uint32_t) * o->list_cap);
    }
    for (uint32_t i = 0; i < rl->n_nodes; ++i) {
        const uint32_t t = o->n_list++;
        o->row[t] = rl->row[i]; o->node_id[t] = rl->node_id[i]; o->base_id[t] = rl->base_id[i]; o->md_row[t] = rl->md_row[i];
        if (failed_out) failed_out[i] = 0;
        const uint32_t row = rl->row[i], md = rl->md_row[i];
        orc_vector_data x;
        x.code = (const uint8_t *)g->codes + (size_t)row * cb;
        x.mag = g->mags[row];
        x.has_id = 1;
        x.id = rl->base_id[i];
        x.md_bits = md == ORC_EMPTY ? NULL : mg->md_bits + (size_t)md * mg->md_dims;
        x.md_mag = md == ORC_EMPTY ? 0.0f : mg->md_mags[md];
        const int under_pseudo = x.md_bits && x.md_mag != 0.0f;
        const uint32_t max_level = rl->max_level[i];
        uint32_t entry = under_pseudo ? mg->pseudo_entry : g->entry, parent = ORC_EMPTY;
        int failed = 0;
        for (int level = (int)num_levels; level >= 0; --level) {
            blevel *l = &b->lv[level];
            md_refresh_view(b);
            memset(fs, 0, sizeof(uint64_t) * l->nb);
            fs_insert(fs, l->nb, rl->node_id[i]);
            mitem *zl = z + 64 * level;
            uint32_t cnt = 0;
            int rc = traverse_md(mg, (uint32_t)level, entry, &x, ef_construction, shortlist, 64, fs, zl, &cnt, NULL, NULL);
            if (rc == ORC_OK && cnt == 0) {
                orc_vector_data x0 = x, y;
                x0.has_id = 0;
                node_data(mg, (uint32_t)level, entry, &y);
                float d = 0.0f;
                rc = orc_distance_md(g->metric, g->storage_type, g->dim, mg->md_dims, &x0, &y, &d);
                zl[0] = (mitem){mkey(mg, d, y.id), entry, d};
                cnt = 1;
            }
            if (rc != ORC_OK) { failed = 1; break; }
            zn[level] = cnt;
            const uint32_t next_entry = level > 0 ? l->child[zl[0].node] : 0;
            if ((uint32_t)level <= max_level) {
                lv_reserve(l, l->cnt + 1);
                const uint32_t idx = l->cnt++;
                lv_init_node(b->min_key, l, idx, row);
                l->node_id[idx] = rl->node_id[i];
                l->node_md[idx] = md;
                ins_reserve(o, (uint32_t)level);
                o->ins[level][idx] = t;
                if (parent != ORC_EMPTY) b->lv[level + 1].child[parent] = idx;
                node_at[level] = idx;
                parent = idx;
            }
            entry = next_entry;
        }
        if (failed) {
            if (failed_out) failed_out[i] = 1;
            continue;
        }
        const uint32_t top = max_level < num_levels ? max_level : num_levels;
        for (uint32_t level = 0; level <= top; ++level)
            md_create_node_edges(b, &b->lv[level], node_at[level], z + 64 * level, zn[level]);
    }
    md_refresh_view(b);
    free(fs); free(z); free(zn); free(node_at);
}

static int mdo_remove_by_id(blevel *l, uint32_t node, uint32_t id) { /* remove_neighbor_by_id: lowest_index stays stale */
    for (uint32_t s = 0; s < l->nb; ++s)
        if (l->adj[(size_t)node * l->nb + s] == id) { l->adj[(size_t)node * l->nb + s] = ORC_EMPTY; return 1; }
    return 0;
}
static int mdo_is_empty(const blevel *l, uint32_t node) {
    for (uint32_t s = 0; s < l->nb; ++s)
        if (l->adj[(size_t)node * l->nb + s] != ORC_EMPTY) return 0;
    return 1;
}
static int mdo_dead(const blevel *l, uint32_t node, uint32_t r) { return node >= 2 && l->node_row[node] == r; }

/* the relink of an emptied node N: the results minus D, N and the row's nodes, rescored with the replica arms
 * (calculate(N, candidate)), sorted best first (ties: smaller id), through create_node_edges with the replica rules */
static int mdo_relink(mdo *o, uint32_t L, uint32_t N, uint32_t D, const mitem *res, uint32_t nres, uint32_t r) {
    orc_md_built *b = o->b;
    orc_md_graph *mg = &b->mg;
    blevel *l = &b->lv[L];
    mitem cand[DEL_KEEP];
    uint32_t m = 0;
    orc_vector_data x, y;
    node_data(mg, L, N, &x);
    for (uint32_t i = 0; i < nres; ++i) {
        const uint32_t c = res[i].node;
        if (c == D || c == N || mdo_dead(l, c, r)) continue;
        node_data(mg, L, c, &y);
        float d = 0.0f;
        const int rc = orc_distance_md(mg->g.metric, mg->g.storage_type, mg->g.dim, mg->md_dims, &x, &y, &d);
        if (rc != ORC_OK) return rc;
        cand[m++] = (mitem){mkey(mg, d, y.id), c, d};
    }
    qsort(cand, m, sizeof(mitem), cmp_desc);
    md_create_node_edges(b, l, N, cand, m);
    return ORC_OK;
}

/* deletes rows[0..n) one at a time.  deleted[vector rows] is the caller's deletion mask (read and updated).
 * out_status[i]: 0 deleted, 1 already deleted, 2 deleted but an Err hit one of the row's nodes. */
void mdo_delete_rows(mdo *o, const uint32_t *rows, uint32_t n, uint32_t shortlist, uint8_t *deleted, uint8_t *out_status) {
    orc_md_built *b = o->b;
    orc_md_graph *mg = &b->mg;
    orc_graph *g = &mg->g;
    const uint32_t L1 = g->num_levels + 1;
    md_refresh_view(b);
    uint32_t maxnb = 0, maxcnt = 0;
    for (uint32_t L = 0; L < L1; ++L) {
        if (b->lv[L].nb > maxnb) maxnb = b->lv[L].nb;
        if (b->lv[L].cnt > maxcnt) maxcnt = b->lv[L].cnt;
    }
    uint64_t *fs = (uint64_t *)malloc(sizeof(uint64_t) * maxnb);
    uint32_t *tmin = (uint32_t *)malloc(sizeof(uint32_t) * (maxcnt ? maxcnt : 1));
    uint32_t *items = (uint32_t *)malloc(sizeof(uint32_t) * (o->n_list ? o->n_list : 1));
    const size_t cb = orc_code_bytes(g->storage_type, g->dim);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t r = rows[i];
        if (deleted[r]) { out_status[i] = 1; continue; }
        deleted[r] = 1;
        out_status[i] = 0;
        uint32_t ni = 0;
        for (uint32_t t = 0; t < o->n_list; ++t)
            if (o->row[t] == r) items[ni++] = t;
        if (!ni) continue;   /* not in the graph: only marked */
        mitem *res = (mitem *)malloc(sizeof(mitem) * (size_t)ni * L1 * DEL_KEEP);
        uint32_t *zn = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)ni * L1);
        uint32_t *loc = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)ni * L1);
        /* phase A: every item against the graph as of the row's start */
        for (uint32_t k = 0; k < ni; ++k) {
            const uint32_t t = items[k], md = o->md_row[t];
            orc_vector_data x;
            x.code = (const uint8_t *)g->codes + (size_t)r * cb;
            x.mag = g->mags[r];
            x.has_id = 1;
            x.id = o->node_id[t];
            x.md_bits = md == ORC_EMPTY ? NULL : mg->md_bits + (size_t)md * mg->md_dims;
            x.md_mag = md == ORC_EMPTY ? 0.0f : mg->md_mags[md];
            uint32_t entry = x.md_bits && x.md_mag != 0.0f ? mg->pseudo_entry : g->entry;
            int err = 0;
            for (int level = (int)g->num_levels; level >= 0; --level) {
                const blevel *l = &b->lv[level];
                uint32_t *z = zn + (size_t)k * L1 + level;
                loc[(size_t)k * L1 + level] = ORC_EMPTY;
                for (uint32_t j = 2; j < l->cnt; ++j)
                    if (o->ins[level][j] == t) { loc[(size_t)k * L1 + level] = j; break; }
                if (err) { *z = ORC_EMPTY; continue; }
                memset(fs, 0, sizeof(uint64_t) * l->nb);
                uint32_t cnt = 0;
                if (traverse_md(mg, (uint32_t)level, entry, &x, DEL_EF, shortlist, DEL_KEEP, fs, res + ((size_t)k * L1 + level) * DEL_KEEP,
                                &cnt, NULL, NULL) != ORC_OK) {
                    err = 1;   /* D3: no relinks on this level or below */
                    out_status[i] = 2;
                    *z = ORC_EMPTY;
                    continue;
                }
                *z = cnt;
                if (level > 0) entry = l->child[res[((size_t)k * L1 + level) * DEL_KEEP].node];
            }
        }
        for (uint32_t L = 0; L < L1; ++L) {
            blevel *l = &b->lv[L];
            /* the row's nodes, in list order: their own slots (D1), then isolated (D4) */
            for (uint32_t k = 0; k < ni; ++k) {
                const uint32_t D = loc[(size_t)k * L1 + L], z = zn[(size_t)k * L1 + L];
                if (D == ORC_EMPTY) continue;
                const mitem *rs = res + ((size_t)k * L1 + L) * DEL_KEEP;
                for (uint32_t s = 0; s < l->nb; ++s) {
                    const uint32_t N = l->adj[(size_t)D * l->nb + s];
                    if (N == ORC_EMPTY) continue;
                    if (mdo_remove_by_id(l, N, D) && !mdo_dead(l, N, r) && mdo_is_empty(l, N) && z != ORC_EMPTY &&
                        mdo_relink(o, L, N, D, rs, z, r) != ORC_OK)
                        out_status[i] = 2;
                }
                for (uint32_t s = 0; s < l->nb; ++s) l->adj[(size_t)D * l->nb + s] = ORC_EMPTY;
                l->lowest_idx[D] = 0;
                l->lowest_key[D] = b->min_key;
            }
            /* D2: links to the row's nodes from outside their lists; a touched node takes the first item it named */
            for (uint32_t x = 0; x < l->cnt; ++x) {
                tmin[x] = ORC_EMPTY;
                for (uint32_t s = 0; s < l->nb; ++s) {
                    const uint32_t v = l->adj[(size_t)x * l->nb + s];
                    if (v == ORC_EMPTY || !mdo_dead(l, v, r)) continue;
                    l->adj[(size_t)x * l->nb + s] = ORC_EMPTY;
                    uint32_t k = 0;
                    while (loc[(size_t)k * L1 + L] != v) ++k;
                    if (tmin[x] == ORC_EMPTY || k < tmin[x]) tmin[x] = k;
                }
            }
            for (uint32_t x = 0; x < l->cnt; ++x) {
                const uint32_t k = tmin[x];
                if (k == ORC_EMPTY || mdo_dead(l, x, r) || !mdo_is_empty(l, x) || zn[(size_t)k * L1 + L] == ORC_EMPTY) continue;
                if (mdo_relink(o, L, x, loc[(size_t)k * L1 + L], res + ((size_t)k * L1 + L) * DEL_KEEP, zn[(size_t)k * L1 + L], r) != ORC_OK)
                    out_status[i] = 2;
            }
        }
        free(res); free(zn); free(loc);
    }
    free(fs); free(tmin); free(items);
}

const orc_md_graph *mdo_graph(const mdo *o) { return &o->b->mg; }
uint32_t mdo_count(const mdo *o, uint32_t level) { return o->b->lv[level].cnt; }

/* copies of `level`'s arrays (any pointer may be NULL): per node node_row, child, node_id, node_md, lowest_idx, lowest_key,
 * list position; per slot adj, simkey */
void mdo_export(const mdo *o, uint32_t level, uint32_t *node_row, uint32_t *child, uint32_t *node_id, uint32_t *node_md,
                uint32_t *lowest_idx, uint32_t *lowest_key, uint32_t *ins, uint32_t *adj, uint32_t *simkey) {
    const blevel *l = &o->b->lv[level];
    const size_t c = l->cnt, s = (size_t)l->cnt * l->nb;
    if (node_row) memcpy(node_row, l->node_row, c * 4);
    if (child) memcpy(child, l->child, c * 4);
    if (node_id) memcpy(node_id, l->node_id, c * 4);
    if (node_md) memcpy(node_md, l->node_md, c * 4);
    if (lowest_idx) memcpy(lowest_idx, l->lowest_idx, c * 4);
    if (lowest_key) memcpy(lowest_key, l->lowest_key, c * 4);
    if (ins) memcpy(ins, o->ins[level], c * 4);
    if (adj) memcpy(adj, l->adj, s * 4);
    if (simkey) memcpy(simkey, l->simkey, s * 4);
}

/* MetricResult order keys of n scores (to compare slot scores read from the GPU with simkey) */
void mdo_order_keys(int metric, const float *in, uint32_t *out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = orc_order_key(metric, in[i]);
}

/* calculate(x, y) for every filled slot of `level` of a replica graph: x is the slot's node, except on a Pseudo-Metadata
 * edge where x is the Metadata end (the arms are not symmetric there; the builder scores from the Metadata side).
 * out[slot] = the score, rc[slot] = ORC_OK or the Err; empty slots: rc = -1. */
void mdo_slot_calc(const orc_md_graph *mg, uint32_t level, float *out, int *rc) {
    const uint32_t cnt = mg->g.cnt[level], nb = mg_nbrs(mg, level);
    for (uint32_t a = 0; a < cnt; ++a)
        for (uint32_t s = 0; s < nb; ++s) {
            const size_t t = (size_t)a * nb + s;
            const uint32_t b = mg->g.adj[level][t];
            out[t] = 0.0f;
            rc[t] = -1;
            if (b == ORC_EMPTY) continue;
            orc_vector_data x, y;
            node_data(mg, level, a, &x);
            node_data(mg, level, b, &y);
            if (orc_replica_kind(&x) == ORC_KIND_PSEUDO && orc_replica_kind(&y) == ORC_KIND_METADATA) {
                orc_vector_data tmp = x; x = y; y = tmp;
            }
            rc[t] = orc_distance_md(mg->g.metric, mg->g.storage_type, mg->g.dim, mg->md_dims, &x, &y, out + t);
        }
}
