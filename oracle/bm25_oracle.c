/*
 * bm25_oracle.c — CPU oracle (TEST INFRASTRUCTURE ONLY; see bm25_oracle.h).
 *
 * Restates, in plain C, the reference's BM25 arithmetic, sealed-segment index
 * semantics and Block-max WAND top-k search.  Compile with -ffp-contract=off:
 * the reference is Rust, which never fuses a*b+c, and parity is bitwise in f64.
 */
#include "bm25_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define DOC_MAX 0xFFFFFFFFu
#define BLOCK 128

/* ------------------------------------------------------------------------- */
/* fieldnorm codec — crates/bm25/src/bm25.rs:15-283.  The 256-entry table is
 * 0..=40 step 1, then groups of 8 values whose step doubles per group
 * (2,4,8,...), ending at 2_013_265_944; generated here, pinned against the
 * reference's literal table in tests/golden/fieldnorm_table.json. */
static uint32_t g_fn_table[256];
static int g_fn_ready = 0;

static void fn_init(void) {
    if (g_fn_ready) return;
    uint32_t v = 0;
    int n = 0;
    for (; n <= 40; n++) g_fn_table[n] = (uint32_t)n;
    v = 40;
    uint32_t step = 2;
    while (n < 256) {
        for (int i = 0; i < 8 && n < 256; i++) {
            v += step;
            g_fn_table[n++] = v;
        }
        step *= 2;
    }
    g_fn_ready = 1;
}

/* bm25.rs:274-276 */
uint32_t orc_fieldnorm_to_length(uint8_t fieldnorm) {
    fn_init();
    return g_fn_table[fieldnorm];
}

/* bm25.rs:278-283: binary_search; Ok(i) → i, Err(i) → i-1 (largest entry <= length) */
uint8_t orc_length_to_fieldnorm(uint32_t length) {
    fn_init();
    int lo = 0, hi = 256; /* first index with table > length */
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (g_fn_table[mid] <= length) lo = mid + 1;
        else hi = mid;
    }
    return (uint8_t)(lo - 1);
}

/* bm25.rs:285-289 */
double orc_idf(uint32_t n_docs, uint32_t df) {
    double n = (double)n_docs;
    double t = (double)df;
    return log((n + 1.0) / (t + 0.5));
}

/* bm25.rs:291-295 */
double orc_tf(uint8_t fieldnorm, uint32_t tf, double k1, double b, double avgdl) {
    double t = (double)tf;
    double dl = (double)orc_fieldnorm_to_length(fieldnorm);
    return (t * (k1 + 1.0)) / (t + k1 * (1.0 - b + b * dl / avgdl));
}

/* bm25.rs:340-354 */
void orc_cache_new(uint32_t n_docs, uint32_t df, double k1, double b, double avgdl, double *s0,
                   double *s1) {
    *s0 = orc_idf(n_docs, df) * (k1 + 1.0);
    for (int f = 0; f < 256; f++) {
        double dl = (double)orc_fieldnorm_to_length((uint8_t)f);
        s1[f] = k1 * (1.0 - b + b * dl / avgdl);
    }
}

/* bm25.rs:355-358 */
double orc_cache_evaluate(double s0, const double *s1, uint8_t fieldnorm, uint32_t tf) {
    double t = (double)tf;
    return (t * s0) / (t + s1[fieldnorm]);
}

/* crates/score/src/lib.rs:46-52 */
int64_t orc_score_from_f64(double v) {
    int64_t bits;
    memcpy(&bits, &v, 8);
    uint64_t mask = ((uint64_t)(bits >> 63)) >> 1;
    return bits ^ (int64_t)mask;
}

/* crates/score/src/lib.rs:54-60 */
double orc_score_to_f64(int64_t s) {
    uint64_t mask = ((uint64_t)(s >> 63)) >> 1;
    int64_t bits = s ^ (int64_t)mask;
    double v;
    memcpy(&v, &bits, 8);
    return v;
}

/* ------------------------------------------------------------------------- */
/* Index: flush.rs:40-158 restated over flat arrays (no pages, no codec). */

typedef struct {
    uint32_t min_doc, max_doc; /* SummaryTuple, tuples.rs:900-910 */
    uint8_t n;                 /* 1..=128 (128 stored as 128) */
    uint8_t wand_fn;
    uint32_t wand_tf;
    uint64_t first; /* posting index of the block's first posting (stands for wptr_block) */
} orc_summary;

struct orc_index {
    uint32_t n_docs, n_terms;
    uint64_t n_post;
    uint64_t sum_len;
    double k1, b, avgdl;
    uint8_t *fieldnorm;      /* [n_docs] DocumentTuple.fieldnorm */
    const uint64_t *post_off; /* [n_terms+1]  BORROWED from the caller (10 GB at C3: no copy) */
    const uint32_t *post_doc; /* [n_post]     BORROWED */
    const uint32_t *post_tf;  /* [n_post]     BORROWED */
    uint32_t *df;            /* TokenTuple.number_of_documents */
    uint8_t *tok_wand_fn;    /* TokenTuple.wand_fieldnorm */
    uint32_t *tok_wand_tf;   /* TokenTuple.wand_term_frequency */
    uint64_t *sum_off;       /* [n_terms+1] into summaries */
    orc_summary *summaries;
};

/* Wand, bm25.rs:297-332 */
typedef struct {
    double tf;
    uint8_t fn;
    uint32_t term_frequency;
} wand_t;
static void wand_new(wand_t *w) {
    w->tf = 0.0;
    w->fn = 255;
    w->term_frequency = 0;
}
static void wand_push(wand_t *w, uint8_t fn, uint32_t tfv, double k1, double b, double avgdl) {
    double t = orc_tf(fn, tfv, k1, b, avgdl);
    if (w->tf < t) {
        w->tf = t;
        w->fn = fn;
        w->term_frequency = tfv;
    }
}
static void wand_extend(wand_t *w, const wand_t *o) {
    if (w->tf < o->tf) *w = *o;
}

orc_index *orc_index_build(uint32_t n_docs, const uint32_t *doc_len, uint32_t n_terms,
                           const uint64_t *post_off, const uint32_t *post_doc,
                           const uint32_t *post_tf, double k1, double b) {
    fn_init();
    if (n_docs == 0 || n_docs == DOC_MAX) return NULL;
    orc_index *ix = (orc_index *)calloc(1, sizeof(*ix));
    ix->n_docs = n_docs;
    ix->n_terms = n_terms;
    ix->n_post = post_off[n_terms];
    ix->k1 = k1;
    ix->b = b;
    ix->fieldnorm = (uint8_t *)malloc(n_docs);
    /* flush.rs:52-64: N, Σlen use exact lengths; per-doc norm is quantised */
    uint64_t sum = 0;
    for (uint32_t d = 0; d < n_docs; d++) {
        sum += doc_len[d];
        ix->fieldnorm[d] = orc_length_to_fieldnorm(doc_len[d]);
    }
    ix->sum_len = sum;
    ix->avgdl = (double)sum / (double)n_docs; /* flush.rs:66 */
    ix->post_off = post_off;
    ix->post_doc = post_doc;
    ix->post_tf = post_tf;
    ix->df = (uint32_t *)calloc(n_terms ? n_terms : 1, sizeof(uint32_t));
    ix->tok_wand_fn = (uint8_t *)calloc(n_terms ? n_terms : 1, 1);
    ix->tok_wand_tf = (uint32_t *)calloc(n_terms ? n_terms : 1, sizeof(uint32_t));
    ix->sum_off = (uint64_t *)calloc(n_terms + 1, sizeof(uint64_t));
    uint64_t nsum = 0;
    for (uint32_t t = 0; t < n_terms; t++) {
        uint64_t n = post_off[t + 1] - post_off[t];
        ix->sum_off[t] = nsum;
        nsum += (n + BLOCK - 1) / BLOCK;
    }
    ix->sum_off[n_terms] = nsum;
    ix->summaries = (orc_summary *)malloc(sizeof(orc_summary) * (nsum ? nsum : 1));
    int bad = 0;
#pragma omp parallel for schedule(dynamic, 64) reduction(| : bad)
    for (uint32_t t = 0; t < n_terms; t++) {
        uint64_t p0 = post_off[t], p1 = post_off[t + 1];
        wand_t tok;
        wand_new(&tok);
        uint64_t si = ix->sum_off[t];
        uint32_t prev = 0;
        int first = 1;
        /* flush.rs:78-125: blocks of up to 128 consecutive postings of one token */
        for (uint64_t p = p0; p < p1; p += BLOCK) {
            uint64_t e = p + BLOCK < p1 ? p + BLOCK : p1;
            wand_t blk;
            wand_new(&blk);
            for (uint64_t i = p; i < e; i++) {
                uint32_t d = post_doc[i];
                if (d >= n_docs || post_tf[i] == 0 || (!first && d <= prev)) bad = 1;
                if (d >= n_docs) continue;
                prev = d;
                first = 0;
                wand_push(&blk, ix->fieldnorm[d], post_tf[i], k1, b, ix->avgdl);
            }
            wand_extend(&tok, &blk);
            orc_summary *s = &ix->summaries[si++];
            s->min_doc = post_doc[p];
            s->max_doc = post_doc[e - 1];
            s->n = (uint8_t)(e - p);
            s->wand_fn = blk.fn;
            s->wand_tf = blk.term_frequency;
            s->first = p;
        }
        ix->df[t] = (uint32_t)(p1 - p0);
        ix->tok_wand_fn[t] = tok.fn;
        ix->tok_wand_tf[t] = tok.term_frequency;
    }
    if (bad) {
        orc_index_free(ix);
        return NULL;
    }
    return ix;
}

void orc_index_free(orc_index *ix) {
    if (!ix) return;
    free(ix->fieldnorm);
    free(ix->df);
    free(ix->tok_wand_fn);
    free(ix->tok_wand_tf);
    free(ix->sum_off);
    free(ix->summaries);
    free(ix);
}

uint32_t orc_index_n_docs(const orc_index *ix) { return ix->n_docs; }
double orc_index_avgdl(const orc_index *ix) { return ix->avgdl; }
uint32_t orc_index_df(const orc_index *ix, uint32_t t) { return t < ix->n_terms ? ix->df[t] : 0; }
uint8_t orc_index_fieldnorm(const orc_index *ix, uint32_t d) { return ix->fieldnorm[d]; }

/* Query canonicalisation: sort + dedup (datatype/tsvector.rs:96-105), drop
 * unknown terms (search.rs:55-62). Returns count. */
static int cmp_u32(const void *a, const void *b) {
    uint32_t x = *(const uint32_t *)a, y = *(const uint32_t *)b;
    return x < y ? -1 : x > y;
}
static int canon_query(const orc_index *ix, const uint32_t *terms, int n, uint32_t *out) {
    memcpy(out, terms, sizeof(uint32_t) * (size_t)n);
    qsort(out, (size_t)n, sizeof(uint32_t), cmp_u32);
    int m = 0;
    for (int i = 0; i < n; i++) {
        if (i > 0 && out[i] == out[i - 1]) continue;
        if (out[i] >= ix->n_terms || ix->df[out[i]] == 0) continue;
        out[m++] = out[i];
    }
    return m;
}

/* ------------------------------------------------------------------------- */
/* Exhaustive scorer (canonical order). */

typedef struct {
    double s;
    uint32_t d;
} sd_t;
/* "a ranks before b": score desc, doc asc */
static inline int sd_before(const sd_t *a, const sd_t *b) {
    return a->s > b->s || (a->s == b->s && a->d < b->d);
}
static int sd_cmp(const void *pa, const void *pb) {
    const sd_t *a = (const sd_t *)pa, *b = (const sd_t *)pb;
    if (sd_before(a, b)) return -1;
    if (sd_before(b, a)) return 1;
    return 0;
}

int orc_search_exhaustive(const orc_index *ix, const uint32_t *terms, int nterms, int k,
                          const uint8_t *allow, uint32_t *out_doc, double *out_score,
                          uint32_t *tie_group_out) {
    if (tie_group_out) *tie_group_out = 0;
    if (k <= 0 || nterms <= 0) return 0;
    uint32_t *q = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)nterms);
    int m = canon_query(ix, terms, nterms, q);
    uint64_t total = 0;
    for (int j = 0; j < m; j++) total += ix->df[q[j]];
    sd_t *cand = (sd_t *)malloc(sizeof(sd_t) * (total ? total : 1));
    uint64_t nc = 0;
    double s1[256];
    if (m == 1) {
        double s0;
        orc_cache_new(ix->n_docs, ix->df[q[0]], ix->k1, ix->b, ix->avgdl, &s0, s1);
        for (uint64_t p = ix->post_off[q[0]]; p < ix->post_off[q[0] + 1]; p++) {
            uint32_t d = ix->post_doc[p];
            if (allow && !(allow[d >> 3] >> (d & 7) & 1)) continue;
            cand[nc].d = d;
            cand[nc].s = 0.0 + orc_cache_evaluate(s0, s1, ix->fieldnorm[d], ix->post_tf[p]);
            nc++;
        }
    } else if (m > 1) {
        /* m-way merge with cursors; ascending term order inside a doc */
        uint64_t *cur = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)m);
        double *s0 = (double *)malloc(sizeof(double) * (size_t)m);
        for (int j = 0; j < m; j++) {
            cur[j] = ix->post_off[q[j]];
            s0[j] = orc_idf(ix->n_docs, ix->df[q[j]]) * (ix->k1 + 1.0);
        }
        /* s1 depends only on (k1,b,avgdl): identical for every term (bm25.rs:349-352) */
        double dummy;
        orc_cache_new(ix->n_docs, 1, ix->k1, ix->b, ix->avgdl, &dummy, s1);
        for (;;) {
            uint32_t dmin = DOC_MAX;
            for (int j = 0; j < m; j++)
                if (cur[j] < ix->post_off[q[j] + 1] && ix->post_doc[cur[j]] < dmin)
                    dmin = ix->post_doc[cur[j]];
            if (dmin == DOC_MAX) break;
            double s = 0.0;
            for (int j = 0; j < m; j++) {
                if (cur[j] < ix->post_off[q[j] + 1] && ix->post_doc[cur[j]] == dmin) {
                    s += orc_cache_evaluate(s0[j], s1, ix->fieldnorm[dmin], ix->post_tf[cur[j]]);
                    cur[j]++;
                }
            }
            if (allow && !(allow[dmin >> 3] >> (dmin & 7) & 1)) continue;
            cand[nc].d = dmin;
            cand[nc].s = s;
            nc++;
        }
        free(cur);
        free(s0);
    }
    qsort(cand, (size_t)nc, sizeof(sd_t), sd_cmp);
    int n = nc < (uint64_t)k ? (int)nc : k;
    for (int i = 0; i < n; i++) {
        out_doc[i] = cand[i].d;
        out_score[i] = cand[i].s;
    }
    if (tie_group_out && n > 0) {
        uint32_t g = 0;
        for (uint64_t i = 0; i < nc; i++)
            if (cand[i].s == cand[n - 1].s) g++;
        *tie_group_out = g;
    }
    free(cand);
    free(q);
    return n;
}

/* ------------------------------------------------------------------------- */
/* Rust std BinaryHeap restated (max-heap; library/alloc/src/collections/
 * binary_heap/mod.rs — NOT in the reference tree, written from the published
 * algorithm; only matters for the order of equal elements).  Generic over an
 * array of int handles with a user comparator returning <0,0,>0 like Ord::cmp. */

typedef int (*heap_cmp_fn)(const void *ctx, int a, int b);
typedef struct {
    int *data;
    int len, cap;
    heap_cmp_fn cmp;
    const void *ctx;
} bheap;

static void bh_sift_up(bheap *h, int start, int pos) {
    int elt = h->data[pos];
    while (pos > start) {
        int parent = (pos - 1) / 2;
        if (h->cmp(h->ctx, elt, h->data[parent]) <= 0) break;
        h->data[pos] = h->data[parent];
        pos = parent;
    }
    h->data[pos] = elt;
}
static void bh_sift_down_range(bheap *h, int pos, int end) {
    int elt = h->data[pos];
    int child = 2 * pos + 1;
    int lim = end >= 2 ? end - 2 : 0; /* end.saturating_sub(2) */
    while (child <= lim && end >= 2) {
        if (h->cmp(h->ctx, h->data[child], h->data[child + 1]) <= 0) child++;
        if (h->cmp(h->ctx, elt, h->data[child]) >= 0) {
            h->data[pos] = elt;
            return;
        }
        h->data[pos] = h->data[child];
        pos = child;
        child = 2 * pos + 1;
    }
    if (child == end - 1 && h->cmp(h->ctx, elt, h->data[child]) < 0) {
        h->data[pos] = h->data[child];
        pos = child;
    }
    h->data[pos] = elt;
}
static void bh_sift_down_to_bottom(bheap *h, int pos) {
    int end = h->len;
    int start = pos;
    int elt = h->data[pos];
    int child = 2 * pos + 1;
    int lim = end >= 2 ? end - 2 : 0;
    while (child <= lim && end >= 2) {
        if (h->cmp(h->ctx, h->data[child], h->data[child + 1]) <= 0) child++;
        h->data[pos] = h->data[child];
        pos = child;
        child = 2 * pos + 1;
    }
    if (child == end - 1) {
        h->data[pos] = h->data[child];
        pos = child;
    }
    h->data[pos] = elt;
    bh_sift_up(h, start, pos);
}
static void bh_push(bheap *h, int v) {
    if (h->len == h->cap) {
        h->cap = h->cap ? h->cap * 2 : 16;
        h->data = (int *)realloc(h->data, sizeof(int) * (size_t)h->cap);
    }
    int old = h->len;
    h->data[h->len++] = v;
    bh_sift_up(h, 0, old);
}
static int bh_pop(bheap *h) { /* caller checks len > 0 */
    int item = h->data[--h->len];
    if (h->len > 0) {
        int t = h->data[0];
        h->data[0] = item;
        item = t;
        bh_sift_down_to_bottom(h, 0);
    }
    return item;
}
static void bh_rebuild(bheap *h) { /* From<Vec>: heapify */
    int n = h->len / 2;
    while (n > 0) {
        n--;
        bh_sift_down_range(h, n, h->len);
    }
}
static void bh_into_sorted(bheap *h) { /* ascending by cmp, in place */
    int end = h->len;
    while (end > 1) {
        end--;
        int t = h->data[0];
        h->data[0] = h->data[end];
        h->data[end] = t;
        bh_sift_down_range(h, 0, end);
    }
}

/* ------------------------------------------------------------------------- */
/* Results — search.rs:284-314.  Heap of (Reverse<Score>, AlwaysEqual<payload>). */

typedef struct {
    int64_t *score; /* Score(i64) per slot */
    uint32_t *doc;
    int nslots;
    int *freelist;
    int nfree;
    bheap heap;
    int limit;
    int64_t threshold; /* Score */
} results_t;

static int results_cmp(const void *ctx, int a, int b) {
    /* Ord on (Reverse<Score>, AlwaysEqual): Reverse flips; payload never breaks ties */
    const results_t *r = (const results_t *)ctx;
    int64_t x = r->score[a], y = r->score[b];
    return y < x ? -1 : (y > x ? 1 : 0);
}
static void results_init(results_t *r, int limit, double threshold) {
    memset(r, 0, sizeof(*r));
    r->limit = limit;
    r->nslots = limit + 2;
    r->score = (int64_t *)malloc(sizeof(int64_t) * (size_t)r->nslots);
    r->doc = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)r->nslots);
    r->freelist = (int *)malloc(sizeof(int) * (size_t)r->nslots);
    for (int i = 0; i < r->nslots; i++) r->freelist[i] = r->nslots - 1 - i;
    r->nfree = r->nslots;
    r->heap.cmp = results_cmp;
    r->heap.ctx = r;
    r->threshold = orc_score_from_f64(threshold);
}
static void results_free(results_t *r) {
    free(r->score);
    free(r->doc);
    free(r->freelist);
    free(r->heap.data);
}
static inline double results_threshold(const results_t *r) { return orc_score_to_f64(r->threshold); }
/* search.rs:301-310 */
static void results_push(results_t *r, double key, uint32_t doc) {
    int slot = r->freelist[--r->nfree];
    r->score[slot] = orc_score_from_f64(key);
    r->doc[slot] = doc;
    bh_push(&r->heap, slot);
    if (r->heap.len > r->limit) {
        int out = bh_pop(&r->heap);
        r->freelist[r->nfree++] = out;
    }
    if (r->heap.len == r->limit) {
        int64_t top = r->score[r->heap.data[0]];
        if (top > r->threshold) r->threshold = top;
    }
}

/* ------------------------------------------------------------------------- */
/* Cursor — search.rs:316-496 */

typedef struct {
    const orc_index *ix;
    double s0;
    const double *s1;
    double token_ub;
    uint32_t doc;
    uint32_t pos; /* position_in_block */
    uint64_t si, si_end; /* TruncatedTapeReader over the token's summaries */
    orc_summary summary;
    double block_ub;
    int filled;
    orc_wand_stats *st;
} cursor_t;

static inline double cur_eval(const cursor_t *c, uint8_t fn, uint32_t tf) {
    return orc_cache_evaluate(c->s0, c->s1, fn, tf);
}
/* search.rs:484-496 */
static void next_summary(cursor_t *c) {
    if (c->si < c->si_end) {
        c->summary = c->ix->summaries[c->si++];
    } else {
        c->summary.min_doc = DOC_MAX;
        c->summary.max_doc = DOC_MAX;
        c->summary.n = 1;
        c->summary.wand_fn = 255;
        c->summary.wand_tf = 0;
        c->summary.first = 0;
    }
}
/* search.rs:352-396 */
static void cursor_new(cursor_t *c, const orc_index *ix, uint32_t term, double s0,
                       const double *s1, orc_wand_stats *st) {
    c->ix = ix;
    c->s0 = s0;
    c->s1 = s1;
    c->st = st;
    c->token_ub = cur_eval(c, ix->tok_wand_fn[term], ix->tok_wand_tf[term]);
    c->si = ix->sum_off[term];
    c->si_end = ix->sum_off[term + 1];
    next_summary(c);
    c->block_ub = cur_eval(c, c->summary.wand_fn, c->summary.wand_tf);
    c->doc = c->summary.min_doc;
    c->pos = 0;
    c->filled = 0;
}
static inline void cursor_fill(cursor_t *c) {
    if (!c->filled) {
        c->filled = 1;
        if (c->st) {
            c->st->blocks_decoded++;
            c->st->postings_touched += c->summary.n;
        }
    }
}
/* search.rs:412-431 */
static void cursor_seek_block(cursor_t *c, uint32_t doc) {
    if (doc <= c->summary.max_doc) return;
    while (c->summary.max_doc < doc) next_summary(c);
    c->doc = c->summary.min_doc;
    c->pos = 0;
    c->block_ub = cur_eval(c, c->summary.wand_fn, c->summary.wand_tf);
    c->filled = 0;
}
/* search.rs:432-466 */
static void cursor_seek(cursor_t *c, uint32_t doc) {
    cursor_seek_block(c, doc);
    if (doc <= c->doc) return;
    if (doc == c->summary.max_doc) {
        c->doc = c->summary.max_doc;
        c->pos = (uint32_t)c->summary.n - 1;
        return;
    }
    cursor_fill(c);
    const uint32_t *ids = c->ix->post_doc + c->summary.first;
    uint32_t i;
    if (doc == c->doc + 1) {
        i = c->pos + 1;
    } else {
        uint32_t lo = c->pos + 1, hi = c->summary.n; /* binary_search → Ok|Err = lower bound */
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1;
            if (ids[mid] < doc) lo = mid + 1;
            else hi = mid;
        }
        i = lo;
    }
    c->doc = ids[i];
    c->pos = i;
}
/* search.rs:467-481 */
static uint32_t cursor_get(cursor_t *c) {
    cursor_fill(c);
    return c->ix->post_tf[c->summary.first + c->pos];
}

static int cursor_heap_cmp(const void *ctx, int a, int b) {
    /* Ord for Cursor is reversed on document_id (search.rs:345-349) */
    const cursor_t *cs = (const cursor_t *)ctx;
    uint32_t x = cs[a].doc, y = cs[b].doc;
    return y < x ? -1 : (y > x ? 1 : 0);
}

/* search() — search.rs:28-282 (sealed segment only) */
int orc_search_wand(const orc_index *ix, const uint32_t *terms, int nterms, int k,
                    const uint8_t *allow, uint32_t *out_doc, double *out_score,
                    orc_wand_stats *stats) {
    if (k <= 0 || nterms <= 0) return 0;
    uint32_t *q = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)nterms);
    int m = canon_query(ix, terms, nterms, q);
    double s1[256];
    {
        double dummy;
        orc_cache_new(ix->n_docs, 1, ix->k1, ix->b, ix->avgdl, &dummy, s1);
    }
    cursor_t *cs = (cursor_t *)malloc(sizeof(cursor_t) * (size_t)(m ? m : 1));
    for (int j = 0; j < m; j++) {
        double s0 = orc_idf(ix->n_docs, ix->df[q[j]]) * (ix->k1 + 1.0);
        cursor_new(&cs[j], ix, q[j], s0, s1, stats);
    }
    results_t res;
    results_init(&res, k, 0.0); /* search.rs:81 */

    bheap head;
    memset(&head, 0, sizeof(head));
    head.cmp = cursor_heap_cmp;
    head.ctx = cs;
    head.data = (int *)malloc(sizeof(int) * (size_t)(m + 1));
    head.cap = m + 1;
    for (int j = 0; j < m; j++) head.data[j] = j;
    head.len = m;
    bh_rebuild(&head); /* BinaryHeap::from(cursors), search.rs:150 */
    int *tail = (int *)malloc(sizeof(int) * (size_t)(m + 1));
    int ntail = 0;
    int *lead = (int *)malloc(sizeof(int) * (size_t)(m + 1));
    int *fail = (int *)malloc(sizeof(int) * (size_t)(m + 1));

    for (;;) { /* 'main */
        if (stats) stats->pivots++;
        int nlead = 0;
        /* 'lead: search.rs:152-169 */
        {
            double sum = 0.0;
            for (int i = 0; i < ntail; i++) sum += cs[tail[i]].token_ub;
            int found = 0;
            while (head.len > 0) {
                int c = bh_pop(&head);
                if (cs[c].doc == DOC_MAX) goto done;
                if (results_threshold(&res) < sum + cs[c].token_ub) {
                    lead[nlead++] = c;
                    found = 1;
                    break;
                } else {
                    sum += cs[c].token_ub;
                    tail[ntail++] = c;
                }
            }
            if (!found) goto done;
        }
        uint32_t document_id = cs[lead[0]].doc;
        /* search.rs:172-176 */
        while (head.len > 0 && cs[head.data[0]].doc == document_id) lead[nlead++] = bh_pop(&head);
        /* search.rs:177-192: extract_if over tail with seek_block, drained fully */
        {
            int nfail = 0, keep = 0, first_fail = 0;
            for (int i = 0; i < ntail; i++) {
                int c = tail[i];
                cursor_seek_block(&cs[c], document_id);
                if (document_id < cs[c].doc) {
                    fail[nfail++] = c;
                    first_fail = 1;
                } else {
                    tail[keep++] = c;
                }
            }
            if (first_fail) {
                ntail = keep;
                for (int i = 0; i < nlead; i++) bh_push(&head, lead[i]);
                for (int i = 0; i < nfail; i++) bh_push(&head, fail[i]);
                continue;
            }
        }
        /* NOTE: in the reference the seek_block calls on elements after the first
         * failure happen lazily inside `for failure in failures` — the order of
         * seek_block calls is the same (front to back), so the effect is identical. */
        double sum_block_ub = 0.0; /* search.rs:193-202 */
        for (int i = 0; i < ntail; i++) sum_block_ub += cs[tail[i]].block_ub;
        for (int i = 0; i < nlead; i++) sum_block_ub += cs[lead[i]].block_ub;
        if (results_threshold(&res) < sum_block_ub) {
            /* search.rs:204-216: seek tail cursors until the first failure */
            int failed_at = -1;
            for (int i = 0; i < ntail; i++) {
                cursor_seek(&cs[tail[i]], document_id);
                if (document_id < cs[tail[i]].doc) {
                    failed_at = i;
                    break;
                }
            }
            if (failed_at >= 0) {
                int f = tail[failed_at];
                for (int i = failed_at; i + 1 < ntail; i++) tail[i] = tail[i + 1];
                ntail--;
                for (int i = 0; i < nlead; i++) bh_push(&head, lead[i]);
                bh_push(&head, f);
                continue;
            }
            /* search.rs:217-237 */
            uint8_t fn = ix->fieldnorm[document_id];
            int pass = !allow || (allow[document_id >> 3] >> (document_id & 7) & 1);
            if (pass) {
                double result = 0.0;
                for (int i = 0; i < ntail; i++)
                    result += cur_eval(&cs[tail[i]], fn, cursor_get(&cs[tail[i]]));
                for (int i = 0; i < nlead; i++)
                    result += cur_eval(&cs[lead[i]], fn, cursor_get(&cs[lead[i]]));
                results_push(&res, result, document_id);
                if (stats) stats->docs_scored++;
            }
            /* search.rs:238-242 */
            for (int i = 0; i < ntail; i++) {
                cursor_seek(&cs[tail[i]], 1 + document_id);
                bh_push(&head, tail[i]);
            }
            for (int i = 0; i < nlead; i++) {
                cursor_seek(&cs[lead[i]], 1 + document_id);
                bh_push(&head, lead[i]);
            }
            ntail = 0;
        } else {
            /* search.rs:243-279 */
            uint32_t min_max = DOC_MAX;
            for (int i = 0; i < nlead; i++)
                if (cs[lead[i]].summary.max_doc < min_max) min_max = cs[lead[i]].summary.max_doc;
            for (int i = 0; i < ntail; i++)
                if (cs[tail[i]].summary.max_doc < min_max) min_max = cs[tail[i]].summary.max_doc;
            uint32_t peek = head.len > 0 ? cs[head.data[0]].doc : DOC_MAX;
            uint32_t seek_doc = (uint32_t)(1 + min_max); /* min_max < MAX here: lead is live */
            if (peek < seek_doc) seek_doc = peek;
            /* argmax of token_ub, lead scanned before tail, first max wins */
            double mx = -INFINITY;
            int which = 0, at = 0;
            for (int i = 0; i < nlead; i++)
                if (cs[lead[i]].token_ub > mx) {
                    mx = cs[lead[i]].token_ub;
                    which = 0;
                    at = i;
                }
            for (int i = 0; i < ntail; i++)
                if (cs[tail[i]].token_ub > mx) {
                    mx = cs[tail[i]].token_ub;
                    which = 1;
                    at = i;
                }
            int c;
            if (which == 0) {
                c = lead[at];
                for (int i = at; i + 1 < nlead; i++) lead[i] = lead[i + 1];
                nlead--;
            } else {
                c = tail[at];
                for (int i = at; i + 1 < ntail; i++) tail[i] = tail[i + 1];
                ntail--;
            }
            cursor_seek(&cs[c], seek_doc);
            bh_push(&head, c);
            for (int i = 0; i < nlead; i++) bh_push(&head, lead[i]);
        }
    }
done:;
    /* search.rs:281, 311-313: into_sorted_vec ascending by (Reverse<Score>) = best first */
    bh_into_sorted(&res.heap);
    int n = res.heap.len;
    for (int i = 0; i < n; i++) {
        int slot = res.heap.data[i];
        out_doc[i] = res.doc[slot];
        out_score[i] = orc_score_to_f64(res.score[slot]);
    }
    results_free(&res);
    free(head.data);
    free(tail);
    free(lead);
    free(fail);
    free(cs);
    free(q);
    return n;
}

void orc_search_wand_batch(const orc_index *ix, int nq, const uint32_t *q_off,
                           const uint32_t *q_terms, int k, int nthreads, uint32_t *out_doc,
                           double *out_score, uint32_t *out_n, orc_wand_stats *stats_sum) {
    orc_wand_stats tot;
    memset(&tot, 0, sizeof(tot));
#ifdef _OPENMP
    if (nthreads < 1) nthreads = 1;
#pragma omp parallel num_threads(nthreads)
#endif
    {
        orc_wand_stats st;
        memset(&st, 0, sizeof(st));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4)
#endif
        for (int i = 0; i < nq; i++) {
            out_n[i] = (uint32_t)orc_search_wand(ix, q_terms + q_off[i],
                                                 (int)(q_off[i + 1] - q_off[i]), k, NULL,
                                                 out_doc + (size_t)i * (size_t)k,
                                                 out_score + (size_t)i * (size_t)k, &st);
        }
#ifdef _OPENMP
#pragma omp critical
#endif
        {
            tot.docs_scored += st.docs_scored;
            tot.blocks_decoded += st.blocks_decoded;
            tot.postings_touched += st.postings_touched;
            tot.pivots += st.pivots;
        }
    }
    if (stats_sum) *stats_sum = tot;
}

void orc_search_exhaustive_batch(const orc_index *ix, int nq, const uint32_t *q_off,
                                 const uint32_t *q_terms, int k, int nthreads,
                                 uint32_t *out_doc, double *out_score, uint32_t *out_n) {
#ifdef _OPENMP
    if (nthreads < 1) nthreads = 1;
#pragma omp parallel for schedule(dynamic, 4) num_threads(nthreads)
#endif
    for (int i = 0; i < nq; i++) {
        out_n[i] = (uint32_t)orc_search_exhaustive(
            ix, q_terms + q_off[i], (int)(q_off[i + 1] - q_off[i]), k, NULL,
            out_doc + (size_t)i * (size_t)k, out_score + (size_t)i * (size_t)k, NULL);
    }
}

/* evaluate() — evaluate.rs:22-74 */
double orc_evaluate(const orc_index *ix, const uint32_t *doc_terms, const uint32_t *doc_tfs,
                    int doc_n, const uint32_t *query_terms, int query_n) {
    /* Document::length(): saturating Σ tf (vector.rs:77-83) */
    uint64_t len64 = 0;
    for (int i = 0; i < doc_n; i++) {
        len64 += doc_tfs[i];
        if (len64 > 0xFFFFFFFFull) len64 = 0xFFFFFFFFull;
    }
    uint8_t fn = orc_length_to_fieldnorm((uint32_t)len64);
    int cursor = 0;
    double result = 0.0;
    for (int qi = 0; qi < query_n; qi++) {
        uint32_t key = query_terms[qi];
        while (cursor < doc_n && doc_terms[cursor] < key) cursor++;
        if (!(cursor < doc_n && doc_terms[cursor] == key)) continue;
        uint32_t value = doc_tfs[cursor];
        if (key >= ix->n_terms || ix->df[key] == 0) continue; /* address_tokens::read → None */
        double idf = orc_idf(ix->n_docs, ix->df[key]);
        double tf = orc_tf(fn, value, ix->k1, ix->b, ix->avgdl);
        result += idf * tf;
    }
    return result;
}

/* ------------------------------------------------------------------------- */
/* Growing segment (search.rs:83-135): the documents inserted since the last seal are scanned one by one; each is
 * scored with the SEALED segment's statistics — Cache::new(number_of_documents, token.number_of_documents, k1, b,
 * avgdl) of the sealed JumpTuple/TokenTuple (search.rs:49-51,66-77) — over the query tokens that exist in the sealed
 * segment (others are dropped, search.rs:60-62), elements in ascending key order (search.rs:112-118), deleted
 * documents skipped (search.rs:110), pushed only when `threshold() < result` with the initial threshold 0.0
 * (search.rs:81,119).  Exhaustive + canonical order (score desc, growing ordinal asc), like orc_search_exhaustive.
 * Document g: elements elem_term/elem_tf[elem_off[g] .. elem_off[g+1]) (term ordinals ascending; ordinals unknown to
 * the sealed segment, e.g. 0xFFFFFFFF, never match), norm fieldnorm[g]. */
int orc_search_growing(const orc_index *ix, uint32_t n_growing, const uint8_t *fieldnorm, const uint8_t *deleted,
                       const uint64_t *elem_off, const uint32_t *elem_term, const uint32_t *elem_tf,
                       const uint32_t *terms, int nterms, int k, const uint8_t *allow, uint32_t *out_doc,
                       double *out_score) {
    if (k <= 0 || nterms <= 0) return 0;
    uint32_t *q = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)nterms);
    const int m = canon_query(ix, terms, nterms, q); /* tokens found in the sealed segment, ascending */
    double *s0 = (double *)malloc(sizeof(double) * (size_t)(m ? m : 1));
    double s1[256], dummy;
    orc_cache_new(ix->n_docs, 1, ix->k1, ix->b, ix->avgdl, &dummy, s1);
    for (int j = 0; j < m; j++) s0[j] = orc_idf(ix->n_docs, ix->df[q[j]]) * (ix->k1 + 1.0);
    sd_t *cand = (sd_t *)malloc(sizeof(sd_t) * (n_growing ? n_growing : 1));
    uint64_t nc = 0;
    for (uint32_t g = 0; g < n_growing && m > 0; g++) {
        if (deleted && deleted[g]) continue;
        double result = 0.0;
        for (uint64_t e = elem_off[g]; e < elem_off[g + 1]; e++) {
            /* tokens.binary_search_by_key(&key) */
            int lo = 0, hi = m;
            while (lo < hi) {
                int mid = (lo + hi) >> 1;
                if (q[mid] < elem_term[e]) lo = mid + 1;
                else hi = mid;
            }
            if (lo < m && q[lo] == elem_term[e]) result += orc_cache_evaluate(s0[lo], s1, fieldnorm[g], elem_tf[e]);
        }
        if (!(0.0 < result)) continue; /* results.threshold() < result */
        if (allow && !(allow[g >> 3] >> (g & 7) & 1)) continue;
        cand[nc].d = g;
        cand[nc].s = result;
        nc++;
    }
    qsort(cand, (size_t)nc, sizeof(sd_t), sd_cmp);
    const int n = nc < (uint64_t)k ? (int)nc : k;
    for (int i = 0; i < n; i++) {
        out_doc[i] = cand[i].d;
        out_score[i] = cand[i].s;
    }
    free(cand);
    free(s0);
    free(q);
    return n;
}

/* ------------------------------------------------------------------------- */
/* Synthetic corpus spec (SURVEY §8d; mirrors tests/fuzz:168-205: L draws with
 * replacement, duplicates aggregated into tf, doc length = L).  Counter-based
 * so any doc can be regenerated independently on CPU or GPU. */

uint64_t orc_splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    uint64_t z = x;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

uint64_t orc_draw(uint64_t seed, uint64_t item, uint32_t j) {
    uint64_t h = orc_splitmix64(seed ^ orc_splitmix64(item));
    return orc_splitmix64(h + (uint64_t)j * 0x9E3779B97F4A7C15ull);
}

void orc_zipf_thresholds(uint32_t vocab, double s, uint64_t *thr) {
    /* thr[r] = floor(2^64 * CDF(r)), CDF cumulative over weights (r+1)^-s */
    double total = 0.0;
    for (uint32_t r = 0; r < vocab; r++) total += pow((double)(r + 1), -s);
    double acc = 0.0;
    for (uint32_t r = 0; r < vocab; r++) {
        acc += pow((double)(r + 1), -s);
        double c = acc / total;
        if (c >= 1.0 || r + 1 == vocab) thr[r] = 0xFFFFFFFFFFFFFFFFull;
        else thr[r] = (uint64_t)ldexp(c, 64);
    }
}

uint32_t orc_draw_term(uint64_t u, uint32_t vocab, const uint64_t *zipf_thr) {
    if (!zipf_thr) return (uint32_t)(((u >> 32) * (uint64_t)vocab) >> 32);
    uint32_t lo = 0, hi = vocab - 1; /* first r with u <= thr[r] */
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (u <= zipf_thr[mid]) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

/* ascending sort of n term ids: LSD radix, 11 bits per pass (the generator's inner loop: qsort() with a callback
 * was 80 % of the corpus generation time) */
static void sort_terms(uint32_t *v, uint32_t *tmp, uint32_t n, uint32_t vocab) {
    if (n < 2) return;
    uint32_t *src = v, *dst = tmp;
    for (uint32_t shift = 0; shift < 32 && (shift == 0 || (vocab - 1) >> shift); shift += 11) {
        uint32_t cnt[2049];
        memset(cnt, 0, sizeof cnt);
        for (uint32_t i = 0; i < n; i++) cnt[((src[i] >> shift) & 2047u) + 1]++;
        for (uint32_t b = 0; b < 2048; b++) cnt[b + 1] += cnt[b];
        for (uint32_t i = 0; i < n; i++) dst[cnt[(src[i] >> shift) & 2047u]++] = src[i];
        uint32_t *t = src;
        src = dst;
        dst = t;
    }
    if (src != v) memcpy(v, src, sizeof(uint32_t) * n);
}

int orc_synth_doc(uint64_t seed, uint32_t doc, uint32_t vocab, uint32_t len_min,
                  uint32_t len_max, const uint64_t *zipf_thr, uint32_t *terms_out,
                  uint32_t *tfs_out, uint32_t *len_out) {
    uint32_t L = len_min;
    if (len_max > len_min) {
        uint64_t u = orc_draw(seed, doc, 0xFFFFFFFFu);
        L = len_min + (uint32_t)(((u >> 32) * (uint64_t)(len_max - len_min + 1)) >> 32);
    }
    uint32_t stack_buf[2 * 512];
    uint32_t *tmp = L <= 512 ? stack_buf : (uint32_t *)malloc(sizeof(uint32_t) * 2 * (size_t)L);
    for (uint32_t j = 0; j < L; j++) tmp[j] = orc_draw_term(orc_draw(seed, doc, j), vocab, zipf_thr);
    sort_terms(tmp, tmp + L, L, vocab);
    int n = 0;
    for (uint32_t j = 0; j < L; j++) {
        if (n > 0 && terms_out[n - 1] == tmp[j]) tfs_out[n - 1]++;
        else {
            terms_out[n] = tmp[j];
            tfs_out[n] = 1;
            n++;
        }
    }
    if (tmp != stack_buf) free(tmp);
    *len_out = L;
    return n;
}

/* SummaryTuple.{wand_fieldnorm, wand_term_frequency} of every block, in (token, block) order — what flush() stores
 * next to min/max_document_id (flush.rs:101-120, tuples.rs:900-910). */
void orc_index_block_wand(const orc_index *ix, uint8_t *fn_out, uint32_t *tf_out) {
    const uint64_t n = ix->sum_off[ix->n_terms];
    for (uint64_t i = 0; i < n; i++) {
        fn_out[i] = ix->summaries[i].wand_fn;
        tf_out[i] = ix->summaries[i].wand_tf;
    }
}
uint64_t orc_index_n_blocks(const orc_index *ix) { return ix->sum_off[ix->n_terms]; }
