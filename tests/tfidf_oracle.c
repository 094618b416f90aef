/* tfidf_oracle.c -- CPU restatement of the reference's TF-IDF / BM25 index (TEST INFRASTRUCTURE ONLY), line by line:
 *   TFIDFIndex::insert / mark_embedding_as_deleted   src/indexes/tf_idf/mod.rs:85-137 (N = total_documents_count)
 *   TFIDFIndexRoot::insert / delete                  src/models/tf_idf_index.rs:315-352 (a list per term hash)
 *   VersionedVec push / push_sorted / delete / len / iter   src/models/versioned_vec.rs:106-275
 *   SparseAnnQueryBasic::search_bm25, get_idf        src/models/sparse_ann_query.rs:149-302
 *   BinaryHeap push / pop (Rust std: sift_up with a `<=` break; pop = swap-remove, sift_down_to_bottom taking the right
 *   child when left <= right, then sift_up), PostingListHead ordered by reversed doc id.
 * A list word is kept as (id, tf bits, state) instead of the reference's packed u64; comparisons use the id the packed
 * word reads as (u32::MAX for a marked entry, 1 << 31 | inserted version for a tombstone), so for ids < 2^31 it is the
 * reference's list word for word.  Ids >= 2^31, which the reference reads as tombstones, are searched here like any other.
 * Two summation modes:
 *   mode 0 (query): a document's products in the caller's query-term order (the GPU contract);
 *   mode 1 (heap):  in the reference's heap pop order.  A query with an empty head among two or more heads makes the
 *                   reference panic (unreachable! in PostingListHead::cmp); here such heads are left out and the query
 *                   is flagged.
 * Built with -ffp-contract=off: every product and sum is rounded on its own. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { LIVE = 0, MARKED = 1, TOMB = 2 };
typedef struct { uint32_t id; uint32_t tf_bits; uint32_t state; } Word;
typedef struct { uint32_t version; uint32_t n, cap; Word *w; } Seg;
typedef struct { uint32_t hash; uint32_t nseg; Seg *segs; } Term;

typedef struct {
    uint32_t id_base;
    uint32_t documents;                 /* total_documents_count */
    uint32_t nterms, tcap;
    Term *terms;                        /* ascending hash */
    uint64_t nrows, rcap, npairs, pcap;
    uint64_t *row_off;
    uint32_t *hashes;
    uint8_t *counted, *deleted;
} TO;

static uint32_t eff_id(const Word *w) {
    if (w->state == MARKED) return 0xFFFFFFFFu;
    if (w->state == TOMB) return 0x80000000u | w->tf_bits;   /* tombstone: tf_bits holds the inserted version */
    return w->id;
}

static Seg *seg_for(Term *t, uint32_t version) {   /* the chain's segment of `version`, appended if missing */
    for (uint32_t i = 0; i < t->nseg; ++i)
        if (t->segs[i].version == version) return &t->segs[i];
    t->segs = realloc(t->segs, (t->nseg + 1) * sizeof(Seg));
    Seg *s = &t->segs[t->nseg++];
    s->version = version;
    s->n = s->cap = 0;
    s->w = NULL;
    return s;
}

static void seg_insert(Seg *s, uint32_t at, Word w) {
    if (s->n == s->cap) { s->cap = s->cap ? 2 * s->cap : 4; s->w = realloc(s->w, s->cap * sizeof(Word)); }
    memmove(s->w + at + 1, s->w + at, (s->n - at) * sizeof(Word));
    s->w[at] = w;
    s->n++;
}

static void push_sorted(Term *t, uint32_t version, uint32_t id, uint32_t tf_bits) {
    Seg *s = seg_for(t, version);
    uint32_t i = s->n;
    while (i > 0 && eff_id(&s->w[i - 1]) > id) --i;
    Word w = {id, tf_bits, LIVE};
    seg_insert(s, i, w);
}

static void vv_delete(Term *t, uint32_t version, uint32_t id) {
    /* find_and_mark_deleted: the first word reading as `id`, in chain order */
    uint32_t ins_version = 0, idx = 0;
    int found = 0;
    for (uint32_t i = 0; i < t->nseg && !found; ++i)
        for (uint32_t j = 0; j < t->segs[i].n; ++j)
            if (t->segs[i].w[j].state == LIVE && t->segs[i].w[j].id == id) {
                t->segs[i].w[j].state = MARKED;
                ins_version = t->segs[i].version;
                idx = j;
                found = 1;
                break;
            }
    if (!found) return;
    /* delete_internal */
    Seg *s = seg_for(t, version);
    if (ins_version == version) {
        memmove(s->w + idx, s->w + idx + 1, (s->n - idx - 1) * sizeof(Word));
        s->n--;
    } else {
        Word w = {0, ins_version, TOMB};
        seg_insert(s, s->n, w);
    }
}

static uint32_t vv_len(const Term *t) {
    uint32_t n = 0;
    for (uint32_t i = 0; i < t->nseg; ++i) n += t->segs[i].n;
    return n;
}

static Term *find_term(const TO *o, uint32_t hash) {
    uint32_t lo = 0, hi = o->nterms;
    while (lo < hi) { const uint32_t m = (lo + hi) / 2; if (o->terms[m].hash < hash) lo = m + 1; else hi = m; }
    return lo < o->nterms && o->terms[lo].hash == hash ? &o->terms[lo] : NULL;
}

static float get_idf(uint32_t documents_count, uint32_t documents_containing_term) {
    return log1pf(((float)(uint32_t)(documents_count - documents_containing_term) + 0.5f) / ((float)documents_containing_term + 0.5f));
}

TO *to_create(uint32_t id_base) {
    TO *o = calloc(1, sizeof(TO));
    o->id_base = id_base;
    o->rcap = 16;
    o->row_off = calloc(o->rcap + 1, 8);
    o->counted = calloc(o->rcap, 1);
    o->deleted = calloc(o->rcap, 1);
    return o;
}

void to_destroy(TO *o) {
    for (uint32_t i = 0; i < o->nterms; ++i) {
        for (uint32_t j = 0; j < o->terms[i].nseg; ++j) free(o->terms[i].segs[j].w);
        free(o->terms[i].segs);
    }
    free(o->terms); free(o->row_off); free(o->hashes); free(o->counted); free(o->deleted);
    free(o);
}

static int cmp_u32(const void *a, const void *b) {
    const uint32_t x = *(const uint32_t *)a, y = *(const uint32_t *)b;
    return x < y ? -1 : x > y;
}

/* n rows (CSR), counted[r] (NULL = all), inserted at `version` */
void to_append(TO *o, const uint64_t *row_off, const uint32_t *hashes, const float *tfs, const uint8_t *counted, uint64_t n,
               uint32_t version) {
    const uint64_t np = row_off[n];
    /* the new terms, merged into the ascending table */
    uint32_t *nh = malloc((np ? np : 1) * 4);
    uint64_t nn = 0;
    for (uint64_t p = 0; p < np; ++p)
        if (!find_term(o, hashes[p])) nh[nn++] = hashes[p];
    qsort(nh, nn, 4, cmp_u32);
    uint64_t u = 0;
    for (uint64_t i = 0; i < nn; ++i)
        if (u == 0 || nh[u - 1] != nh[i]) nh[u++] = nh[i];
    if (u) {
        o->terms = realloc(o->terms, (o->nterms + u) * sizeof(Term));
        int64_t i = (int64_t)o->nterms - 1, j = (int64_t)u - 1, k = (int64_t)(o->nterms + u) - 1;
        while (j >= 0) {
            if (i >= 0 && o->terms[i].hash > nh[j]) o->terms[k--] = o->terms[i--];
            else { Term t = {nh[j--], 0, NULL}; o->terms[k--] = t; }
        }
        o->nterms += (uint32_t)u;
    }
    free(nh);
    /* rows */
    while (o->nrows + n > o->rcap) {
        o->rcap *= 2;
        o->row_off = realloc(o->row_off, (o->rcap + 1) * 8);
        o->counted = realloc(o->counted, o->rcap);
        o->deleted = realloc(o->deleted, o->rcap);
    }
    if (o->npairs + np > o->pcap) {
        o->pcap = (o->npairs + np) * 2;
        o->hashes = realloc(o->hashes, o->pcap * 4);
    }
    memcpy(o->hashes + o->npairs, hashes, np * 4);
    for (uint64_t r = 0; r < n; ++r) {
        const uint64_t row = o->nrows + r;
        o->row_off[row + 1] = o->npairs + row_off[r + 1];
        o->counted[row] = counted ? counted[r] != 0 : 1;
        o->deleted[row] = 0;
        if (o->counted[row]) o->documents += 1;     /* total_documents_count.fetch_add(1) */
        const uint32_t id = o->id_base + (uint32_t)row;
        for (uint64_t p = row_off[r]; p < row_off[r + 1]; ++p) {
            uint32_t bits;
            memcpy(&bits, &tfs[p], 4);
            push_sorted(find_term(o, hashes[p]), version, id, bits);
        }
    }
    o->nrows += n;
    o->npairs += np;
}

/* deletes rows[0..n) at `version`; a deleted row again is a no-op */
void to_delete(TO *o, const uint32_t *rows, uint64_t n, uint32_t version) {
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t r = rows[i];
        if (o->deleted[r]) continue;
        o->deleted[r] = 1;
        if (!o->counted[r]) continue;             /* delete_embedding: no text, nothing to do */
        o->documents -= 1;                        /* total_documents_count.fetch_sub(1) */
        for (uint64_t p = o->row_off[r]; p < o->row_off[r + 1]; ++p)
            vv_delete(find_term(o, o->hashes[p]), version, o->id_base + r);
    }
}

/* -> N; df / idf per hash (absent: df 0, idf NaN) */
uint32_t to_term_stats(const TO *o, const uint32_t *hashes, uint64_t n, uint32_t *out_df, float *out_idf) {
    for (uint64_t i = 0; i < n; ++i) {
        const Term *t = find_term(o, hashes[i]);
        out_df[i] = t ? vv_len(t) : 0;
        out_idf[i] = t ? get_idf(o->documents, out_df[i]) : nanf("");
    }
    return o->documents;
}

/* ---------------------------------------------------------------- heads */
typedef struct { const Term *t; uint32_t seg, pos; float idf; } Head;

static void head_skip(Head *h) {   /* VersionedVecIter: skip marked and tombstone words, then the next segment */
    while (h->seg < h->t->nseg) {
        const Seg *s = &h->t->segs[h->seg];
        while (h->pos < s->n && s->w[h->pos].state != LIVE) h->pos++;
        if (h->pos < s->n) return;
        h->seg++;
        h->pos = 0;
    }
}
static int head_live(const Head *h) { return h->seg < h->t->nseg; }
static const Word *head_peek(const Head *h) { return &h->t->segs[h->seg].w[h->pos]; }
static void head_next(Head *h) { h->pos++; head_skip(h); }

/* a <= b in PostingListHead's Ord (o.0.cmp(&s.0)): a's doc id >= b's */
static int le(const Head *a, const Head *b) { return head_peek(a)->id >= head_peek(b)->id; }

typedef struct { Head **d; uint32_t n; } Heap;
static void sift_up(Heap *hp, uint32_t start, uint32_t pos) {
    Head *e = hp->d[pos];
    while (pos > start) {
        const uint32_t parent = (pos - 1) / 2;
        if (le(e, hp->d[parent])) break;
        hp->d[pos] = hp->d[parent];
        pos = parent;
    }
    hp->d[pos] = e;
}
static void heap_push(Heap *hp, Head *h) { hp->d[hp->n++] = h; sift_up(hp, 0, hp->n - 1); }
static void sift_down_to_bottom(Heap *hp, uint32_t pos) {
    const uint32_t end = hp->n, start = pos;
    Head *e = hp->d[pos];
    uint32_t child = 2 * pos + 1;
    while (child <= (end >= 2 ? end - 2 : 0)) {
        child += le(hp->d[child], hp->d[child + 1]) ? 1 : 0;
        hp->d[pos] = hp->d[child];
        pos = child;
        child = 2 * pos + 1;
    }
    if (child == end - 1) { hp->d[pos] = hp->d[child]; pos = child; }
    hp->d[pos] = e;
    sift_up(hp, start, pos);
}
static Head *heap_pop(Heap *hp) {
    if (!hp->n) return NULL;
    Head *item = hp->d[--hp->n];
    if (hp->n) { Head *t = hp->d[0]; hp->d[0] = item; item = t; sift_down_to_bottom(hp, 0); }
    return item;
}

static float f32_of(uint32_t bits) { float f; memcpy(&f, &bits, 4); return f; }

/* scores of one query over every row: acc[r] valid where touched[r]; matches[r] = products added; abssum[r] = sum of
 * |product| (double).  Returns 1 if the reference would panic on this query (heap mode only). */
int to_scores(const TO *o, int mode, const uint32_t *q, uint64_t nq, float *acc, uint8_t *touched, uint32_t *matches,
              double *abssum) {
    memset(touched, 0, o->nrows);
    if (matches) memset(matches, 0, o->nrows * 4);
    if (abssum) memset(abssum, 0, o->nrows * 8);
    Head *heads = malloc((nq ? nq : 1) * sizeof(Head));
    uint32_t nh = 0, empty = 0;
    for (uint64_t j = 0; j < nq; ++j) {
        const Term *t = find_term(o, q[j]);
        if (!t) continue;
        Head h = {t, 0, 0, get_idf(o->documents, vv_len(t))};
        head_skip(&h);
        if (!head_live(&h)) { ++empty; continue; }
        heads[nh++] = h;
    }
    const int panic = mode == 1 && empty && nh + empty >= 2;
#define ADD(row, prod)                                                           \
    do {                                                                         \
        const float p_ = (prod);                                                 \
        if (touched[row]) acc[row] = acc[row] + p_; else { acc[row] = p_; touched[row] = 1; } \
        if (matches) matches[row]++;                                             \
        if (abssum) abssum[row] += fabs((double)p_);                             \
    } while (0)
    if (mode == 0) {
        for (uint32_t i = 0; i < nh; ++i)
            for (Head h = heads[i]; head_live(&h); head_next(&h)) {
                const Word *w = head_peek(&h);
                ADD(w->id - o->id_base, f32_of(w->tf_bits) * h.idf);
            }
    } else {
        Heap hp = {malloc((nh ? nh : 1) * sizeof(Head *)), 0};
        for (uint32_t i = 0; i < nh; ++i) heap_push(&hp, &heads[i]);
        Head *head;
        while ((head = heap_pop(&hp))) {
            if (!head_live(head)) continue;
            const uint32_t doc = head_peek(head)->id;
            const float tf = f32_of(head_peek(head)->tf_bits);
            head_next(head);
            const uint32_t row = doc - o->id_base;
            ADD(row, tf * head->idf);
            if (head_live(head)) heap_push(&hp, head);
            while (hp.n) {
                Head *top = hp.d[0];
                if (!head_live(top)) { heap_pop(&hp); continue; }
                if (head_peek(top)->id != doc) break;
                ADD(row, f32_of(head_peek(top)->tf_bits) * top->idf);
                Head *h2 = heap_pop(&hp);
                head_next(h2);
                if (head_live(h2)) heap_push(&hp, h2);
            }
        }
        free(hp.d);
    }
#undef ADD
    free(heads);
    return panic;
}

static uint32_t total_key(float v) {   /* f32::total_cmp as an unsigned key */
    uint32_t b;
    memcpy(&b, &v, 4);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
typedef struct { uint32_t key; uint32_t id; float s; } Ranked;
static int cmp_ranked(const void *a, const void *b) {
    const Ranked *x = a, *y = b;
    if (x->key != y->key) return x->key > y->key ? -1 : 1;
    return x->id < y->id ? -1 : x->id > y->id;
}

/* queries as CSR of hashes; out_ids / out_scores [nq][kout] (kout = k == 0 || k > 512 ? 512 : k), out_counts [nq],
 * out_panic [nq] (may be NULL) */
void to_search(const TO *o, int mode, const uint64_t *q_off, const uint32_t *q_hashes, uint32_t nq, uint32_t k, uint32_t *out_ids,
               float *out_scores, uint32_t *out_counts, uint8_t *out_panic) {
    const uint32_t kout = (k == 0 || k > 512) ? 512 : k;
#pragma omp parallel for schedule(dynamic, 1)
    for (uint32_t q = 0; q < nq; ++q) {
        float *acc = malloc((o->nrows ? o->nrows : 1) * 4);
        uint8_t *touched = malloc(o->nrows ? o->nrows : 1);
        const int panic = to_scores(o, mode, q_hashes + q_off[q], q_off[q + 1] - q_off[q], acc, touched, NULL, NULL);
        if (out_panic) out_panic[q] = (uint8_t)panic;
        /* the buckets, docs visited in ascending id (the heap pops the smallest id first) */
        uint32_t bid[512];
        float bs[512];
        for (int b = 0; b < 512; ++b) { bid[b] = 0xFFFFFFFFu; bs[b] = -INFINITY; }
        for (uint64_t r = 0; r < o->nrows; ++r) {
            if (!touched[r]) continue;
            const uint32_t id = o->id_base + (uint32_t)r, b = id % 512;
            if (acc[r] > bs[b]) { bs[b] = acc[r]; bid[b] = id; }
        }
        Ranked rk[512];
        uint32_t n = 0;
        for (int b = 0; b < 512; ++b)
            if (bid[b] != 0xFFFFFFFFu) { rk[n].key = total_key(bs[b]); rk[n].id = bid[b]; rk[n].s = bs[b]; ++n; }
        qsort(rk, n, sizeof(Ranked), cmp_ranked);
        const uint32_t cnt = n < kout ? n : kout;
        for (uint32_t i = 0; i < kout; ++i) {
            out_ids[(size_t)q * kout + i] = i < cnt ? rk[i].id : 0xFFFFFFFFu;
            out_scores[(size_t)q * kout + i] = i < cnt ? rk[i].s : 0.0f;
        }
        out_counts[q] = cnt;
        free(acc);
        free(touched);
    }
}

float to_idf(uint32_t documents_count, uint32_t df) { return get_idf(documents_count, df); }
uint64_t to_rows(const TO *o) { return o->nrows; }
