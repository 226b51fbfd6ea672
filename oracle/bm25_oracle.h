/*
 * bm25_oracle.h — CPU oracle for the BM25 top-k hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (vectorchord-bm25_b200/)
 * may include, link or call this.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs use it, as the checker and
 * as the timed CPU baseline, never as the thing shipped.
 *
 * It is a plain-C restatement of the reference's algorithm (Rust, not
 * buildable here: no rustc/cargo/Postgres).  Every function cites the
 * reference file:line it follows (paths relative to the reference tree).
 *
 * Parity pins: the fieldnorm table, Score bit trick, the sqllogictest ranking
 * goldens and hand-checked Cache::evaluate values are pinned in
 * tests/test_oracle_golden.py.  Golden *scores* are pinned nowhere in the
 * reference (it has no unit tests in crates/bm25), and the order of equal
 * scores in the reference is decided by Rust std BinaryHeap internals
 * (toolchain unpinned): TIE ORDER IS PARITY-UNPINNED; the canonical rule
 * used everywhere here is (score desc, doc id asc).
 */
#ifndef BM25_ORACLE_H
#define BM25_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- crates/bm25/src/bm25.rs:15-283 fieldnorm codec ---- */
uint32_t orc_fieldnorm_to_length(uint8_t fieldnorm);
uint8_t orc_length_to_fieldnorm(uint32_t length);
/* ---- crates/bm25/src/bm25.rs:285-295 ---- */
double orc_idf(uint32_t n_docs, uint32_t df);
double orc_tf(uint8_t fieldnorm, uint32_t tf, double k1, double b, double avgdl);
/* ---- crates/bm25/src/bm25.rs:334-359 Cache ---- */
void orc_cache_new(uint32_t n_docs, uint32_t df, double k1, double b, double avgdl,
                   double *s0, double *s1_256);
double orc_cache_evaluate(double s0, const double *s1_256, uint8_t fieldnorm, uint32_t tf);
/* ---- crates/score/src/lib.rs:46-60 ---- */
int64_t orc_score_from_f64(double v);
double orc_score_to_f64(int64_t s);

/* ---- sealed-segment index: restatement of flush.rs:40-158 over flat arrays ---- */
typedef struct orc_index orc_index;

/* Build from a term-major CSR corpus (doc ids ascending inside a term, tf != 0).
 * doc_len[d] is the exact document length (Σ tf, vector.rs:77-83).
 * The three posting arrays are BORROWED (not copied): keep them alive until orc_index_free.
 * Returns NULL on invalid input. */
orc_index *orc_index_build(uint32_t n_docs, const uint32_t *doc_len, uint32_t n_terms,
                           const uint64_t *post_off, const uint32_t *post_doc,
                           const uint32_t *post_tf, double k1, double b);
void orc_index_free(orc_index *idx);
uint32_t orc_index_n_docs(const orc_index *idx);
double orc_index_avgdl(const orc_index *idx);
uint32_t orc_index_df(const orc_index *idx, uint32_t term);
uint8_t orc_index_fieldnorm(const orc_index *idx, uint32_t doc);

/* Exhaustive f64 scorer with the canonical order (score desc, doc asc).
 * terms[] need not be sorted/deduped; unknown terms (>= n_terms or df == 0) are
 * dropped (search.rs:60-62).  Per-doc sum runs over query terms in ascending
 * term order with Cache::evaluate (bm25.rs:355-358).  allow = optional bitmap
 * (bit d set → doc d passes the filter, search.rs:230); NULL = all pass.
 * If tie_group_out != NULL it receives the number of docs whose score equals
 * the k-th returned score (>= 1 when k results are returned; for tie-aware checks).
 * Returns number of results (<= k). */
int orc_search_exhaustive(const orc_index *idx, const uint32_t *terms, int nterms, int k,
                          const uint8_t *allow, uint32_t *out_doc, double *out_score,
                          uint32_t *tie_group_out);

typedef struct {
    uint64_t docs_scored;      /* results.push calls (search.rs:236) */
    uint64_t blocks_decoded;   /* fill_block calls (search.rs:498) */
    uint64_t postings_touched; /* 128 per decoded full block, n per tail block */
    uint64_t pivots;           /* 'main iterations */
} orc_wand_stats;

/* Block-max WAND restatement of search() (search.rs:28-282) over the in-memory
 * index (no growing segment: benchmarks have none, search.rs:83-135 is skipped).
 * Output order = Results::into_sorted_vec (search.rs:311-313) with a restated
 * std BinaryHeap, so equal scores come out in heap order, NOT canonical order. */
int orc_search_wand(const orc_index *idx, const uint32_t *terms, int nterms, int k,
                    const uint8_t *allow, uint32_t *out_doc, double *out_score,
                    orc_wand_stats *stats);

/* Batch drivers for timing (OpenMP over queries when nthreads > 1).
 * q_off[nq+1] indexes q_terms.  out arrays are nq*k, out_n is nq. */
void orc_search_wand_batch(const orc_index *idx, int nq, const uint32_t *q_off,
                           const uint32_t *q_terms, int k, int nthreads, uint32_t *out_doc,
                           double *out_score, uint32_t *out_n, orc_wand_stats *stats_sum);
void orc_search_exhaustive_batch(const orc_index *idx, int nq, const uint32_t *q_off,
                                 const uint32_t *q_terms, int k, int nthreads,
                                 uint32_t *out_doc, double *out_score, uint32_t *out_n);

/* evaluate() for the <&> operator path (evaluate.rs:22-74): document given as
 * sorted distinct (term, tf); query as sorted distinct terms.  Positive score
 * (the SQL wrapper negates, operators.rs:54). */
double orc_evaluate(const orc_index *idx, const uint32_t *doc_terms, const uint32_t *doc_tfs,
                    int doc_n, const uint32_t *query_terms, int query_n);

/* Growing segment scan (search.rs:83-135) against the sealed index `idx`: exhaustive, canonical order; doc ids are
 * growing ordinals.  Returns the number of results (<= k). */
int orc_search_growing(const orc_index *idx, uint32_t n_growing, const uint8_t *fieldnorm, const uint8_t *deleted,
                       const uint64_t *elem_off, const uint32_t *elem_term, const uint32_t *elem_tf,
                       const uint32_t *terms, int nterms, int k, const uint8_t *allow, uint32_t *out_doc,
                       double *out_score);

/* SummaryTuple.{wand_fieldnorm, wand_term_frequency} of every 128-posting block, (token, block) order (flush.rs:101-120) */
void orc_index_block_wand(const orc_index *idx, uint8_t *fn_out, uint32_t *tf_out);
uint64_t orc_index_n_blocks(const orc_index *idx);

/* ---- synthetic corpus spec (ours, SURVEY §8d; mirrors tests/fuzz:168-205) ---- */
uint64_t orc_splitmix64(uint64_t x);
/* Build the integer inverse-CDF thresholds for Zipf(s) over `vocab` ranks
 * (s == 0 → not used, uniform draw).  thr must hold vocab entries. */
void orc_zipf_thresholds(uint32_t vocab, double s, uint64_t *thr);
/* The j-th raw draw of document (or query) `item` under `seed`. */
uint64_t orc_draw(uint64_t seed, uint64_t item, uint32_t j);
uint32_t orc_draw_term(uint64_t u, uint32_t vocab, const uint64_t *zipf_thr);
/* Generate one document: returns number of distinct terms written (sorted). */
int orc_synth_doc(uint64_t seed, uint32_t doc, uint32_t vocab, uint32_t len_min,
                  uint32_t len_max, const uint64_t *zipf_thr, uint32_t *terms_out,
                  uint32_t *tfs_out, uint32_t *len_out);

/* Bulk forms (bm25_synth.c): the whole corpus as term-major CSR, and a batch of queries. */
int orc_synth_corpus(uint64_t seed, uint32_t n_docs, uint32_t vocab, uint32_t len_min, uint32_t len_max, double zipf_s,
                     int nthreads, uint32_t *doc_len, uint64_t *post_off, uint32_t *post_doc, uint32_t *post_tf,
                     uint64_t cap, uint64_t *n_post_out);
int orc_synth_queries(uint64_t seed, uint32_t nq, uint32_t vocab, uint32_t nmin, uint32_t nmax, double zipf_s,
                      const uint64_t *post_off, uint32_t *q_off, uint32_t *q_terms);

/* ---- posting-block codec (bm25_codec.c): compression.rs:36-136 + crates/simd bit/byte packing ---- */
uint32_t orc_compress_document_ids(uint32_t min_doc, const uint32_t *docs, uint32_t n, uint8_t *meta, uint8_t *out);
uint32_t orc_decompress_document_ids(uint32_t min_doc, uint8_t meta, const uint8_t *in, uint32_t n_bytes,
                                     uint32_t *docs);
uint32_t orc_compress_term_frequencies(const uint32_t *tfs, uint32_t n, uint8_t *meta, uint8_t *out);
uint32_t orc_decompress_term_frequencies(uint8_t meta, const uint8_t *in, uint32_t n_bytes, uint32_t *tfs);
/* flush.rs:78-120 over a CSR corpus: two passes (bytes == NULL → sizes only); returns the payload size */
uint64_t orc_encode_blocks(uint32_t n_terms, const uint64_t *post_off, const uint32_t *post_doc,
                           const uint32_t *post_tf, uint64_t *term_blk_off, uint32_t *blk_min, uint32_t *blk_n,
                           uint8_t *meta_doc, uint8_t *meta_tf, uint64_t *doc_off, uint64_t *tf_off,
                           uint8_t *bytes);

#ifdef __cplusplus
}
#endif
#endif
