/* sparse_oracle.c -- CPU restatement of the reference's sparse inverted index (TEST INFRASTRUCTURE ONLY), line by line:
 *   InvertedIndexNode::quantize            src/models/inverted_index.rs:168-172
 *   SparseAnnQueryBasic::sequential_search  src/models/sparse_ann_query.rs:68-147
 *   finalize_sparse_ann_results            src/indexes/inverted/mod.rs:331-381
 *   sample_embedding / finalize_sampling    src/indexes/inverted/mod.rs:148-247
 * The posting lists are a per-dim list of (row, key) in insertion order; the reference's hash map of dot products is a
 * dense u32 array plus a touched flag (a row is a candidate as soon as a visited list holds it).  The boundary among equal
 * similarities, unspecified in the reference (select_nth_unstable), is: higher similarity, then smaller id.
 * Built with -ffp-contract=off: the re-rank's multiply and add stay separate. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static uint32_t sat_u32(float x, uint32_t hi) {   /* Rust `as` to an unsigned integer: saturating, NaN -> 0 */
    if (!(x > 0.0f)) return 0;
    if (x >= (float)hi) return hi;
    return (uint32_t)x;
}

uint32_t so_quantize(float value, float ub, uint32_t bits) {
    const uint32_t quantization = (1u << bits) - 1;
    const float max_val = (float)quantization;
    float x = (value / ub) * max_val;
    if (x < 0.0f) x = 0.0f;            /* f32::clamp keeps NaN */
    if (x > max_val) x = max_val;
    uint32_t q = sat_u32(x, 255);
    return q < quantization ? q : quantization;
}

void so_thresholds(float thr, uint32_t bits, uint32_t *etv, uint32_t *low) {
    const float p = (float)(1u << bits) * thr;
    const float m = isnan(p) ? 255.0f : (p < 255.0f ? p : 255.0f);   /* f32::min returns the non-NaN operand */
    *etv = sat_u32(m, 255);
    *low = sat_u32(thr * (float)(1u << bits), 0xFFFFFFFFu);
}

typedef struct { uint32_t dim; uint32_t n; uint32_t *row; uint8_t *key; } List;

static int cmp_dim(const void *a, const void *b) {
    const uint32_t x = ((const List *)a)->dim, y = ((const List *)b)->dim;
    return x < y ? -1 : x > y;
}

typedef struct { uint32_t sim; uint32_t id; } Cand;
static int cmp_cand(const void *a, const void *b) {
    const Cand *x = a, *y = b;
    if (x->sim != y->sim) return x->sim > y->sim ? -1 : 1;
    return x->id < y->id ? -1 : x->id > y->id;
}

static uint32_t total_key(float v) {   /* f32::total_cmp as an unsigned key; NaN canonicalised to the sign-set quiet NaN */
    uint32_t b;
    if (v != v) b = 0xFFC00000u;
    else memcpy(&b, &v, 4);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
typedef struct { uint32_t key; uint32_t id; float dp; } Ranked;
static int cmp_ranked(const void *a, const void *b) {
    const Ranked *x = a, *y = b;
    if (x->key != y->key) return x->key > y->key ? -1 : 1;
    return x->id < y->id ? -1 : x->id > y->id;
}

/* n_rows rows as CSR (row_off[n_rows+1], dims, vals); deleted[r] != 0 = tombstoned (may be NULL).  For each of nq queries
 * (CSR q_off / q_dims / q_vals): out_ids / out_scores [nq][k] (CDB_INVALID_ID / 0 in unused slots), out_counts [nq]. */
void so_search(uint32_t bits, float ub, float thr, int rerank, uint32_t factor, uint32_t k, uint32_t id_base, uint64_t n_rows,
               const uint64_t *row_off, const uint32_t *dims, const float *vals, const uint8_t *deleted, uint32_t nq,
               const uint64_t *q_off, const uint32_t *q_dims, const float *q_vals, uint32_t *out_ids, float *out_scores,
               uint32_t *out_counts) {
    const uint32_t one_quantized = (1u << bits) - 1;
    uint32_t etv, low;
    so_thresholds(thr, bits, &etv, &low);
    /* InvertedIndex::insert: every pair of every row goes to the list of its dim under its key */
    const uint64_t np = row_off[n_rows];
    List *tmp = calloc(np ? np : 1, sizeof(List));
    uint64_t nl = 0;
    for (uint64_t p = 0; p < np; ++p) { tmp[p].dim = dims[p]; }
    qsort(tmp, np, sizeof(List), cmp_dim);
    for (uint64_t p = 0; p < np; ++p)
        if (nl == 0 || tmp[nl - 1].dim != tmp[p].dim) tmp[nl++] = tmp[p];
    List *lists = calloc(nl ? nl : 1, sizeof(List));
    memcpy(lists, tmp, nl * sizeof(List));
    free(tmp);
    for (uint64_t r = 0; r < n_rows; ++r)
        for (uint64_t p = row_off[r]; p < row_off[r + 1]; ++p) {
            List key = {dims[p], 0, 0, 0};
            List *l = bsearch(&key, lists, nl, sizeof(List), cmp_dim);
            l->n++;
        }
    for (uint64_t i = 0; i < nl; ++i) {
        lists[i].row = malloc(lists[i].n * 4 + 4);
        lists[i].key = malloc(lists[i].n + 1);
        lists[i].n = 0;
    }
    for (uint64_t r = 0; r < n_rows; ++r)
        for (uint64_t p = row_off[r]; p < row_off[r + 1]; ++p) {
            List key = {dims[p], 0, 0, 0};
            List *l = bsearch(&key, lists, nl, sizeof(List), cmp_dim);
            l->row[l->n] = (uint32_t)r;
            l->key[l->n] = (uint8_t)so_quantize(vals[p], ub, bits);
            l->n++;
        }
    const uint64_t kf = (uint64_t)k * (rerank ? factor : 1);
#pragma omp parallel for schedule(dynamic, 1)
    for (uint32_t q = 0; q < nq; ++q) {
        uint32_t *dot = calloc(n_rows ? n_rows : 1, 4);
        uint8_t *touched = calloc(n_rows ? n_rows : 1, 1);
        for (uint64_t j = q_off[q]; j < q_off[q + 1]; ++j) {
            List key = {q_dims[j], 0, 0, 0};
            const List *l = bsearch(&key, lists, nl, sizeof(List), cmp_dim);
            if (!l) continue;
            const uint32_t qv = so_quantize(q_vals[j], ub, bits);
            /* qv > low: keys max..=0; else keys etv..=max (empty when etv > max) */
            const uint32_t kmin = qv > low ? 0 : etv;
            for (uint32_t i = 0; i < l->n; ++i) {
                const uint32_t kk = l->key[i];
                if (kk < kmin || kk > one_quantized) continue;
                const uint32_t r = l->row[i];
                if (deleted && deleted[r]) continue;
                dot[r] += qv * kk;
                touched[r] = 1;
            }
        }
        uint64_t nc = 0;
        for (uint64_t r = 0; r < n_rows; ++r) nc += touched[r];
        Cand *c = malloc((nc ? nc : 1) * sizeof(Cand));
        nc = 0;
        for (uint64_t r = 0; r < n_rows; ++r)
            if (touched[r]) { c[nc].sim = dot[r]; c[nc].id = id_base + (uint32_t)r; ++nc; }
        qsort(c, nc, sizeof(Cand), cmp_cand);
        if (nc > kf) nc = kf;
        uint32_t cnt = 0;
        if (!rerank) {
            for (; cnt < nc && cnt < k; ++cnt) {
                out_ids[(size_t)q * k + cnt] = c[cnt].id;
                out_scores[(size_t)q * k + cnt] = (float)c[cnt].sim;
            }
        } else {
            Ranked *rk = malloc((nc ? nc : 1) * sizeof(Ranked));
            for (uint64_t i = 0; i < nc; ++i) {
                const uint64_t r = c[i].id - id_base;
                float dp = 0.0f;
                for (uint64_t j = q_off[q]; j < q_off[q + 1]; ++j) {
                    /* HashMap from the row's pairs: the last pair of a dim wins */
                    int found = 0;
                    float val = 0.0f;
                    for (uint64_t p = row_off[r]; p < row_off[r + 1]; ++p)
                        if (dims[p] == q_dims[j]) { val = vals[p]; found = 1; }
                    if (found) dp += val * q_vals[j];
                }
                rk[i].dp = dp;
                rk[i].id = c[i].id;
                rk[i].key = total_key(dp);
            }
            qsort(rk, nc, sizeof(Ranked), cmp_ranked);
            for (; cnt < nc && cnt < k; ++cnt) {
                out_ids[(size_t)q * k + cnt] = rk[cnt].id;
                out_scores[(size_t)q * k + cnt] = rk[cnt].dp != rk[cnt].dp ? -NAN : rk[cnt].dp;
            }
            free(rk);
        }
        for (uint32_t i = cnt; i < k; ++i) { out_ids[(size_t)q * k + i] = 0xFFFFFFFFu; out_scores[(size_t)q * k + i] = 0.0f; }
        out_counts[q] = cnt;
        free(c);
        free(dot);
        free(touched);
    }
    for (uint64_t i = 0; i < nl; ++i) { free(lists[i].row); free(lists[i].key); }
    free(lists);
}

/* counts[t-1] += #values > t (t = 1..9); returns values_upper_bound for values_collected = n_values */
float so_sample(const float *values, uint64_t n, float clamp_margin_percent, const uint64_t *prior, uint64_t prior_values,
                uint64_t *counts) {
    for (int t = 0; t < 9; ++t) counts[t] = prior ? prior[t] : 0;
    for (uint64_t i = 0; i < n; ++i)
        for (int t = 0; t < 9; ++t) counts[t] += values[i] > (float)(t + 1);
    const float values_count = (float)(n + (prior ? prior_values : 0));
    for (int t = 0; t < 9; ++t)
        if (((float)counts[t] / values_count) * 100.0f <= clamp_margin_percent) return (float)(t + 1);
    return 10.0f;
}
