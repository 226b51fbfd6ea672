// bm25x_evaluate.cu — bm25::evaluate (crates/bm25/src/evaluate.rs:22-74), the score behind `<&>` outside an index scan
// (src/index/operators.rs:22-55), for batches of (document, query) pairs (DESIGN §4.2).
//
// One kernel, k_evaluate, serves every entry point: documents and queries as term ordinals (bm25x_evaluate_batch and its
// sharded form), or the rows the tsvector casts leave on the device (bm25x_evaluate_tsvectors and its sharded form).  It
// scores with the statistics it is given: an index's own, or a document-sharded index's whole segment.
#include <math.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "bm25x_build.h"

uint32_t bm25x_fieldnorm_to_length(uint8_t fn);

namespace {

// The statistics of one segment, device arrays: fieldnorm -> length [256], idf [n_terms] (the host libm, like the
// reference's f64::ln), df [n_terms], s1d [256].
struct EvalStats {
    const uint32_t *fn_len;
    const double *idf;
    const uint32_t *df;
    const double *s1d;
    uint32_t n_terms;
    double k1;
};

// One thread per (document, query) pair: pair p scores document row p against query row pair_query[p] (p when NULL).
// Rows are either strictly ascending ordinals, or a cast's rows in key order: the vocabulary is sorted bytewise, so known
// ordinals ascend, with entries >= n_terms (BM25X_TERM_MISSING) interleaved among them on either side.  The merge
// therefore skips a query entry >= n_terms before it moves the document cursor, and steps over document entries
// >= n_terms while it advances; entries >= n_terms are never merged.  On strictly ascending rows those entries sit at the
// tail and the two rules change nothing.
template <typename Off>
__global__ void k_evaluate(uint32_t n_pairs, const Off *__restrict__ d_off, const uint32_t *__restrict__ d_terms,
                           const uint32_t *__restrict__ d_tfs, const Off *__restrict__ q_off,
                           const uint32_t *__restrict__ q_terms, const uint32_t *__restrict__ pair_query,
                           const EvalStats st, double *__restrict__ out) {
    const uint32_t pidx = blockIdx.x * blockDim.x + threadIdx.x;
    if (pidx >= n_pairs) return;
    const uint32_t q = pair_query ? pair_query[pidx] : pidx;
    const Off a = d_off[pidx], b = d_off[pidx + 1];
    uint64_t len = 0;  // Document::length(): saturating Σ tf over the whole row (vector.rs:77-83)
    for (Off i = a; i < b; ++i) {
        len += d_tfs[i];
        if (len > 0xFFFFFFFFull) len = 0xFFFFFFFFull;
    }
    int lo = 0, hi = 256;  // length_to_fieldnorm, bm25.rs:278-283
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (st.fn_len[mid] <= (uint32_t)len) lo = mid + 1;
        else hi = mid;
    }
    const int fn = lo - 1;
    const uint32_t T = st.n_terms;
    Off cursor = a;
    double result = 0.0;
    const double k1p1 = __dadd_rn(st.k1, 1.0);
    for (Off qi = q_off[q], qe = q_off[q + 1]; qi < qe; ++qi) {
        const uint32_t key = q_terms[qi];
        if (key >= T) continue;  // address_tokens::read → None
        while (cursor < b && (d_terms[cursor] < key || d_terms[cursor] >= T)) cursor++;
        if (!(cursor < b && d_terms[cursor] == key) || st.df[key] == 0) continue;
        double tfd = (double)d_tfs[cursor];
        double tfv = __ddiv_rn(__dmul_rn(tfd, k1p1), __dadd_rn(tfd, st.s1d[fn]));  // bm25.rs:291-295
        result = __dadd_rn(result, __dmul_rn(st.idf[key], tfv));
    }
    out[pidx] = result;
}

// idf of every term (bm25.rs:285-289) of a segment of N documents, uploaded to the current device.
cudaError_t upload_idf(uint32_t N, const std::vector<uint32_t> &df, uint32_t T, double **out) {
    std::vector<double> h_idf(T ? T : 1);
    for (uint32_t t = 0; t < T; ++t) h_idf[t] = log(((double)N + 1.0) / ((double)df[t] + 0.5));
    cudaError_t e = cudaMalloc((void **)out, 8 * (size_t)(T ? T : 1));
    if (e == cudaSuccess) e = cudaMemcpy(*out, h_idf.data(), 8 * (size_t)(T ? T : 1), cudaMemcpyHostToDevice);
    return e;
}

// ix's tables, built on first use and kept with the handle: the fieldnorm -> length table, and (with_idf) the idf table,
// which bm25x_index_finalize_replica drops when a refill brings another df.  Leaves ix->device current.
int index_tables(bm25x_index *ix, bool with_idf) {
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    std::lock_guard<std::mutex> lk(ix->eval_mutex);
    if (!ix->eval_fn_len) {
        uint32_t h_fn[256];
        for (int f = 0; f < 256; ++f) h_fn[f] = bm25x_fieldnorm_to_length((uint8_t)f);
        uint32_t *d_fn = nullptr;
        BM25X_CUDA_TRY(cudaMalloc((void **)&d_fn, sizeof(h_fn)));
        ix->allocs.push_back((void *)d_fn);
        BM25X_CUDA_TRY(cudaMemcpy(d_fn, h_fn, sizeof(h_fn), cudaMemcpyHostToDevice));
        ix->eval_fn_len = d_fn;
    }
    if (with_idf && !ix->eval_idf) {
        double *d_idf = nullptr;
        const cudaError_t e = upload_idf(ix->d.n_docs, ix->h_df, ix->d.n_terms, &d_idf);
        if (d_idf) ix->allocs.push_back((void *)d_idf);
        BM25X_CUDA_TRY(e);
        ix->eval_idf = d_idf;
    }
    return BM25X_OK;
}

// What an index scores with: its own N, df, avgdl, k1 and b.
int index_stats(bm25x_index *ix, EvalStats *st) {
    const int rc = index_tables(ix, true);
    if (rc != BM25X_OK) return rc;
    *st = {ix->eval_fn_len, ix->eval_idf, ix->d.df, ix->d.s1d, ix->d.n_terms, ix->k1};
    return BM25X_OK;
}

// What a document-sharded index scores with, on shard 0's device: the whole segment's N and df (sx->h_df) as a df array
// and an idf table, built on first use under sx->eval_mutex and freed by bm25x_sharded_destroy.  Not shard 0's own idf
// table or d.df: those hold the shard's local N and df.  Its s1d is the segment's (every shard is built from one Stats).
int sharded_stats(bm25x_sharded_index *sx, EvalStats *st) {
    bm25x_index *s0 = sx->shards[0];
    int rc = index_tables(s0, false);
    if (rc != BM25X_OK) return rc;
    {
        std::lock_guard<std::mutex> lk(sx->eval_mutex);
        const uint32_t T = sx->n_terms;
        if (!sx->eval_df) {
            uint32_t *d_df = nullptr;
            cudaError_t e = cudaMalloc((void **)&d_df, 4 * (size_t)(T ? T : 1));
            if (e == cudaSuccess && T) e = cudaMemcpy(d_df, sx->h_df.data(), 4 * (size_t)T, cudaMemcpyHostToDevice);
            if (e != cudaSuccess) cudaFree(d_df);
            BM25X_CUDA_TRY(e);
            sx->eval_df = d_df;
        }
        if (!sx->eval_idf) {
            double *d_idf = nullptr;
            const cudaError_t e = upload_idf(sx->n_docs, sx->h_df, T, &d_idf);
            if (e != cudaSuccess) cudaFree(d_idf);
            BM25X_CUDA_TRY(e);
            sx->eval_idf = d_idf;
        }
    }
    *st = {s0->eval_fn_len, sx->eval_idf, sx->eval_df, s0->d.s1d, sx->n_terms, s0->k1};
    return BM25X_OK;
}

// k_evaluate over n_pairs pairs of device rows on the current device (pair_q: device, or NULL), out downloaded.
template <typename Off>
int launch(const char *who, Scratch &sc, uint32_t n_pairs, const Off *d_off, const uint32_t *d_terms,
           const uint32_t *d_tfs, const Off *q_off, const uint32_t *q_terms, const uint32_t *pair_q,
           const EvalStats &st, double *out) {
    double *g_out = sc.alloc<double>(n_pairs);
    if (sc.e == cudaSuccess) {
        k_evaluate<Off><<<(unsigned)(((uint64_t)n_pairs + 127) / 128), 128>>>(n_pairs, d_off, d_terms, d_tfs, q_off,
                                                                             q_terms, pair_q, st, g_out);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(out, g_out, 8 * (size_t)n_pairs, cudaMemcpyDeviceToHost);
    if (sc.e != cudaSuccess) {
        bm25x_set_error("%s: %s", who, cudaGetErrorString(sc.e));
        return BM25X_ERR_CUDA;
    }
    return BM25X_OK;
}

// ---- documents and queries as term ordinals ----

// The host checks of bm25x_evaluate_batch and its sharded form: null arguments, then the Document / Query invariants
// (vector.rs:46-134).  *done: nothing to score.
int check_ordinal_pairs(const char *who, const void *h, uint32_t n_pairs, const uint32_t *d_off, const uint32_t *d_terms,
                        const uint32_t *d_tfs, const uint32_t *q_off, const uint32_t *q_terms, const double *out,
                        bool *done) {
    *done = false;
    if (!h || (n_pairs && (!d_off || !q_off || !out))) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *done = n_pairs == 0;
    if (*done) return BM25X_OK;
    if (d_off[n_pairs] != 0 && !d_tfs) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    int vrc = bm25x_check_vectors(n_pairs, d_off, d_terms, d_tfs);
    if (vrc == BM25X_OK) vrc = bm25x_check_vectors(n_pairs, q_off, q_terms, nullptr);
    return vrc;
}

int evaluate_ordinals(const char *who, int device, const EvalStats &st, uint32_t n_pairs, const uint32_t *d_off,
                      const uint32_t *d_terms, const uint32_t *d_tfs, const uint32_t *q_off, const uint32_t *q_terms,
                      double *out) {
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const uint32_t nd = d_off[n_pairs], nqt = q_off[n_pairs];
    const uint32_t *g_doff = sc.up(d_off, (size_t)n_pairs + 1), *g_dt = sc.up(d_terms, nd), *g_df = sc.up(d_tfs, nd);
    const uint32_t *g_qoff = sc.up(q_off, (size_t)n_pairs + 1), *g_qt = sc.up(q_terms, nqt);
    return launch<uint32_t>(who, sc, n_pairs, g_doff, g_dt, g_df, g_qoff, g_qt, nullptr, st, out);
}

// ---- documents and queries as tsvectors ----

// The host checks of bm25x_evaluate_tsvectors and its sharded form up to the handle's own: null arguments, the document
// tsvectors' refusals in document mode, the queries' in query mode, then pair_query.
int check_tsvector_pairs(const char *who, const void *h, const uint8_t *seed, const bm25x_tsvectors *docs,
                         const bm25x_tsvectors *queries, const uint32_t *pair_query, const double *out) {
    if (!h || !seed || !docs || !queries || (docs->n && !out)) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_tsvectors(who, docs, 0);
    if (rc == BM25X_OK) rc = check_tsvectors(who, queries, 1);
    if (rc != BM25X_OK) return rc;
    if (!pair_query) {
        if (queries->n != docs->n) {
            bm25x_set_error("%s: pair_query is NULL, but there are %u query tsvectors for %u document tsvectors", who,
                            queries->n, docs->n);
            return BM25X_ERR_INVALID;
        }
        return BM25X_OK;
    }
    for (uint32_t p = 0; p < docs->n; p++)
        if (pair_query[p] >= queries->n) {
            bm25x_set_error("%s: pair_query[%u] = %u is not below the %u query tsvectors", who, p, pair_query[p],
                            queries->n);
            return BM25X_ERR_INVALID;
        }
    return BM25X_OK;
}

// Both casts on keys->device against its vocabulary, then k_evaluate with st: only out comes down.  keys: the index, or
// shard 0 of a document-sharded index, which holds the segment's keys and their device copy.
int evaluate_tsvectors(const char *who, bm25x_index *keys, const EvalStats &st, const uint8_t seed[32],
                       const bm25x_tsvectors *docs, const bm25x_tsvectors *queries, const uint32_t *pair_query,
                       double *out) {
    const uint32_t n = docs->n;
    const TsvVocab v{keys->device, &keys->h_keys, keys->d.n_terms, &keys->key_vocab, &keys->key_vocab_mutex};
    TsvCast d(keys->device), q(keys->device);
    int rc = tsvector_cast(who, v, seed, docs, 0, d);  // a merged count of 0 is refused here, before out is written
    if (rc == BM25X_OK) rc = tsvector_cast(who, v, seed, queries, 1, q);
    if (rc != BM25X_OK) return rc;
    Scratch sc(keys->device);
    sc.e = cudaSetDevice(keys->device);
    const uint64_t *g_doff = sc.up(d.off.data(), d.off.size()), *g_qoff = sc.up(q.off.data(), q.off.size());
    const uint32_t *g_pq = pair_query ? sc.up(pair_query, n) : nullptr;
    return launch<uint64_t>(who, sc, n, g_doff, d.ord, d.tf, g_qoff, q.ord, g_pq, st, out);
}

// bm25x_lookup_terms' refusal of a handle without term keys (replicas, keyless builds).
int keyless_refusal(const bm25x_index *ix) {
    if (!ix->h_keys.empty() || !ix->d.n_terms) return BM25X_OK;
    bm25x_set_error("bm25x_lookup_terms: index was created without term keys");
    return BM25X_ERR_INVALID;
}

// The refusals of a handle that bm25::evaluate cannot score with.
int check_index(const char *who, const bm25x_index *ix) {
    if (ix->h_df.size() != ix->d.n_terms) {
        bm25x_set_error("%s: replica not finalized (bm25x_index_finalize_replica)", who);
        return BM25X_ERR_INVALID;
    }
    // bm25::evaluate reads one segment's meta and tokens (evaluate.rs:22-74): a handle whose avgdl is another segment's
    // while its N and df are its own matches no reference answer
    if (!own_statistics(ix)) {
        bm25x_set_error("%s: the index scores with another segment's statistics (a growing handle); "
                        "evaluate on the sealed index",
                        who);
        return BM25X_ERR_INVALID;
    }
    return BM25X_OK;
}

}  // namespace

// Invariants of the reference's vector types (crates/bm25/src/vector.rs:46-134): a Document / Query holds strictly
// ascending keys, a Document's term frequencies are non-zero (`Document::new` / `Query::new` → expect("invalid data")).
// Host only; bm25x_evaluate_batch applies it to both sides of every pair (its kernel merges the two sorted lists).
extern "C" int bm25x_check_vectors(uint32_t n, const uint32_t *off, const uint32_t *terms, const uint32_t *tfs) {
    if (n && (!off || (!terms && off[n] != 0))) {
        bm25x_set_error("bm25x_check_vectors: null argument");
        return BM25X_ERR_INVALID;
    }
    for (uint32_t i = 0; i < n; ++i) {
        if (off[i + 1] < off[i]) {
            bm25x_set_error("invalid data: offsets not monotone at vector %u", i);
            return BM25X_ERR_INVALID;
        }
        for (uint32_t j = off[i]; j < off[i + 1]; ++j) {
            if (j > off[i] && terms[j] <= terms[j - 1]) {
                bm25x_set_error("invalid data: keys of vector %u are not strictly ascending", i);
                return BM25X_ERR_INVALID;
            }
            if (tfs && tfs[j] == 0) {
                bm25x_set_error("invalid data: zero term frequency in vector %u", i);
                return BM25X_ERR_INVALID;
            }
        }
    }
    return BM25X_OK;
}

extern "C" int bm25x_evaluate_batch(bm25x_index *ix, uint32_t n_pairs, const uint32_t *d_off, const uint32_t *d_terms,
                                    const uint32_t *d_tfs, const uint32_t *q_off, const uint32_t *q_terms, double *out) {
    const char *who = "bm25x_evaluate_batch";
    bool done = false;
    int rc = check_ordinal_pairs(who, ix, n_pairs, d_off, d_terms, d_tfs, q_off, q_terms, out, &done);
    if (rc != BM25X_OK || done) return rc;
    rc = check_index(who, ix);
    EvalStats st;
    if (rc == BM25X_OK) rc = index_stats(ix, &st);
    if (rc != BM25X_OK) return rc;
    return evaluate_ordinals(who, ix->device, st, n_pairs, d_off, d_terms, d_tfs, q_off, q_terms, out);
}

extern "C" int bm25x_evaluate_batch_sharded(bm25x_sharded_index *sx, uint32_t n_pairs, const uint32_t *d_off,
                                            const uint32_t *d_terms, const uint32_t *d_tfs, const uint32_t *q_off,
                                            const uint32_t *q_terms, double *out) {
    const char *who = "bm25x_evaluate_batch_sharded";
    bool done = false;
    int rc = check_ordinal_pairs(who, sx, n_pairs, d_off, d_terms, d_tfs, q_off, q_terms, out, &done);
    if (rc != BM25X_OK || done) return rc;
    EvalStats st;
    rc = sharded_stats(sx, &st);
    if (rc != BM25X_OK) return rc;
    return evaluate_ordinals(who, sx->shards[0]->device, st, n_pairs, d_off, d_terms, d_tfs, q_off, q_terms, out);
}

extern "C" int bm25x_evaluate_tsvectors(bm25x_index *ix, const uint8_t seed[32], const bm25x_tsvectors *docs,
                                        const bm25x_tsvectors *queries, const uint32_t *pair_query, double *out) {
    const char *who = "bm25x_evaluate_tsvectors";
    int rc = check_tsvector_pairs(who, ix, seed, docs, queries, pair_query, out);
    if (rc == BM25X_OK) rc = check_index(who, ix);
    if (rc == BM25X_OK) rc = keyless_refusal(ix);
    if (rc != BM25X_OK || docs->n == 0) return rc;
    EvalStats st;
    rc = index_stats(ix, &st);
    if (rc != BM25X_OK) return rc;
    return evaluate_tsvectors(who, ix, st, seed, docs, queries, pair_query, out);
}

extern "C" int bm25x_evaluate_tsvectors_sharded(bm25x_sharded_index *sx, const uint8_t seed[32],
                                                const bm25x_tsvectors *docs, const bm25x_tsvectors *queries,
                                                const uint32_t *pair_query, double *out) {
    const char *who = "bm25x_evaluate_tsvectors_sharded";
    int rc = check_tsvector_pairs(who, sx, seed, docs, queries, pair_query, out);
    if (rc == BM25X_OK) rc = keyless_refusal(sx->shards[0]);
    if (rc != BM25X_OK || docs->n == 0) return rc;
    EvalStats st;
    rc = sharded_stats(sx, &st);
    if (rc != BM25X_OK) return rc;
    return evaluate_tsvectors(who, sx->shards[0], st, seed, docs, queries, pair_query, out);
}
