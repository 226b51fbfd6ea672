// bm25x_build.h — the build contract of every index handle, internal to the library (DESIGN §3).
//
// A builder opens the handle with index_begin (df, statistics, norms, payloads: every array but the postings), writes the
// postings at their padded offsets d.post_off, then calls index_finish_device (pad slots, doc-id copy, block descriptors,
// score bounds, champion lists).  Builders: the CSR builds (bm25x_index.cu), the stored-block ingests (bm25x_blocks.cu),
// the growing segment's create, refresh and seal (bm25x_growing.cu).
#pragma once

#include <functional>
#include <memory>
#include <mutex>
#include <vector>

#include "bm25x_common.h"

namespace {

// Owner of index g in an ascending offset array off[0..n]: the last t with off[t] <= g (the term of a posting, the token of a
// block).
__device__ __forceinline__ uint32_t owner_of(const uint64_t *__restrict__ off, uint32_t n, uint64_t g) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (off[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// Cache::evaluate (bm25.rs:355-358) of term frequency tf in a document of norm fn.  The explicit roundings keep the bits
// of every build kernel the same whatever the compiler contracts.
__device__ __forceinline__ double tf_score(uint32_t tf, uint32_t fn, double s0, const double *__restrict__ s1d) {
    const double tfd = (double)tf;
    return __ddiv_rn(__dmul_rn(tfd, s0), __dadd_rn(tfd, s1d[fn]));
}

// The same of a packed posting word w = tf << 8 | fieldnorm.
__device__ __forceinline__ double posting_score(uint32_t w, double s0, const double *__restrict__ s1d) {
    return tf_score(w >> 8, w & 0xFFu, s0, s1d);
}

// Score bounds are inflated by 2^-40 so that they also dominate any later re-association of the f64 sum.
constexpr double UB_INFLATE = 1.0 + 9.094947017729282e-13;

// A block's bound as stored: the inflated score rounded up to f32.
__device__ __forceinline__ float block_bound(double v) { return __double2float_ru(v * UB_INFLATE); }

}  // namespace

// The statistics a handle scores with: avgdl and the s0 / s1 tables of a segment of N documents with the given df.  The
// only place they are computed is the constructors (bm25x_index.cu): the shards of a segment and its growing segment
// receive the segment's object, so that they score with its bits (DESIGN §4.7).
struct Stats {
    uint64_t sum_len;
    double avgdl;
    std::vector<double> s0d;  // [T]
    std::vector<float> s0f;
    double s1d[256];
    float s1f[256];

    Stats(uint32_t N, uint64_t sum_len, double avgdl, const uint32_t *df, uint32_t T, double k1, double b);
    // a segment's own: avgdl = Σlen / N (flush.rs:52-66)
    Stats(uint32_t N, uint64_t sum_len, const uint32_t *df, uint32_t T, double k1, double b);
};

// Whether a handle scores with its own segment's statistics, avgdl = Σlen / N (flush.rs:52-66).  A handle of
// bm25x_growing_create scores with the sealed segment's avgdl but holds its own documents' N, Σlen and df, and a replica
// of one keeps that avgdl and Σlen through the layout.  The export and the evaluate refuse such handles.
inline bool own_statistics(const bm25x_index *ix) { return ix->avgdl == (double)ix->sum_len / (double)ix->d.n_docs; }

// A half-built handle: an early return destroys it, release() hands it out.
struct IndexDestroy {
    void operator()(bm25x_index *ix) const { bm25x_index_destroy(ix); }
};
using IndexGuard = std::unique_ptr<bm25x_index, IndexDestroy>;

// Device temporaries of one build step on one device, freed when it goes out of scope (every refusal included).  The first
// failure sticks in `e`; later calls do nothing.
struct Scratch {
    int device;
    cudaError_t e = cudaSuccess;
    std::vector<void *> ptrs;
    explicit Scratch(int dev) : device(dev) {}
    Scratch(const Scratch &) = delete;
    ~Scratch() {
        if (ptrs.empty()) return;
        cudaSetDevice(device);
        for (void *p : ptrs) cudaFree(p);
    }
    template <typename T>
    T *alloc(size_t n) {
        T *p = nullptr;
        if (e == cudaSuccess) e = cudaMalloc((void **)&p, sizeof(T) * (n ? n : 1));
        if (e != cudaSuccess) return nullptr;
        ptrs.push_back(p);
        return p;
    }
    template <typename T>
    T *up(const T *h, size_t n) {
        T *p = alloc<T>(n);
        if (e == cudaSuccess && n) e = cudaMemcpy(p, h, sizeof(T) * n, cudaMemcpyHostToDevice);
        return p;
    }
    // p, one of this scratch's allocations, handed to a longer-lived owner that frees it: no longer freed here.
    template <typename T>
    T *release(T *p) {
        ptrs.erase(std::find(ptrs.begin(), ptrs.end(), (void *)p));
        return p;
    }
};

// One handle's documents and terms, from whichever source (CSR columns, reference-format blocks, a shard of either, a
// growing segment).
struct BuildMeta {
    uint32_t n_docs, n_terms;
    const uint32_t *doc_len;
    const uint16_t *payload;
    const uint8_t *term_key;
    double k1, b;
    const uint32_t *df;  // [n_terms]
    uint64_t n_post;
    const uint8_t *fieldnorm = nullptr;  // when doc_len == NULL: DocumentTuple.fieldnorm per doc + JumpTuple.sum_of_document_lengths
    uint64_t sum_len = 0;
    // document shard: global id of local document 0, for the synthesised ctid payload
    uint32_t doc_base = 0;
};

// ---- the build core (bm25x_index.cu) ----

// A handle with everything but the postings, scoring with `given` or, when NULL, its own statistics.
int index_begin(const BuildMeta &m, const Stats *given, int device, IndexGuard &ix);
// After the postings are in place: everything derived from them.
cudaError_t index_finish_device(bm25x_index *ix);
// The postings of a term-major CSR uploaded, then index_finish_device; a CUDA failure is refused as `who`'s.
int upload_csr(bm25x_index *ix, const char *who, uint32_t T, uint64_t P, const uint64_t *post_off,
               const uint32_t *post_doc, const uint32_t *post_tf);

// ---- the build from documents (bm25x_documents.cu) after its host checks: documents c as
// bm25x_index_create_from_documents takes them and has checked them, doc_len[n_docs] their lengths.  The element arrays
// may be device memory on `device` (the tsvector build's cast, bm25x_tsvector.cu); elem_off is host memory.  *out is
// set on success; a CUDA failure is refused as `who`'s.
int documents_build(const char *who, const bm25x_documents *c, const uint32_t *doc_len, int device, bm25x_index **out);
// Its steps, which the sharded build from tsvectors (bm25x_tsvector.cu) runs shard by shard.  vocab_pass: the distinct
// keys of c's elements ascending (host bytes, 16 B each) and each key's count, on `device`.  key_ordinals: term[i] = the
// ordinal in keys[0..T) of raw key i (n 16-byte keys in device memory on `device`, each one of the vocabulary's).
// invert: the postings of documents [lo, hi) of c, local ids, into the handle index_begin opened, then
// index_finish_device; `keys` is read for a keyed c only.
int vocab_pass(const char *who, const bm25x_documents *c, int device, std::vector<uint8_t> &keys,
               std::vector<uint32_t> &df);
cudaError_t key_ordinals(int device, const void *raw, uint64_t n, const std::vector<uint8_t> &keys, uint32_t T,
                         uint32_t *term);
int invert(const char *who, const bm25x_documents *c, const std::vector<uint8_t> &keys, uint32_t lo, uint32_t hi,
           bm25x_index *ix);

// ---- the tsvector casts of a growing segment (bm25x_tsvector.cu) ----

// The host refusals of a batch of tsvectors (bm25x_tsvectors), named by who; as_query: the query cast's.
int check_tsvectors(const char *who, const bm25x_tsvectors *t, int as_query);
// A sealed vocabulary (T sorted 16-byte keys) and where its device copy lives: uploaded to `device` on first use into
// *slot under *mu, freed by the slot's owner.
struct TsvVocab {
    int device;
    const std::vector<uint8_t> *keys;
    uint32_t T;
    void **slot;
    std::mutex *mu;
};
// The cast of a batch on one device (run_cast, bm25x_tsvector.cu).  Outputs held on the device, freed with the object:
// document mode the keyed CSR (raw keys key[E'], tf[E']), query mode the keys, or (a vocabulary given) the keys'
// ordinals ord[E'].  Host: off[n+1] the rows, len[n] the saturating Σ tf of each row (document mode), and the first
// vector with a merged tf of 0 / >= 2^24.
struct TsvCast {
    Scratch sc;
    ulonglong2 *key = nullptr;
    uint32_t *tf = nullptr, *ord = nullptr;
    std::vector<uint64_t> off;
    std::vector<uint32_t> len;
    uint32_t zero = 0xFFFFFFFFu, big = 0xFFFFFFFFu;
    explicit TsvCast(int device) : sc(device) {}
};
// The cast of t (checked) on v.device, left there without keys: c.ord the ordinal of each key in v's vocabulary
// (BM25X_TERM_MISSING where it lacks the key; each row in key order, so known ordinals ascend with BM25X_TERM_MISSING
// among them), c.tf in document mode, and c.off.  Refusals: the cast's (a document element whose merged count is 0, after
// the device work), CUDA failures named by who.  A merged tf >= 2^24 is not refused (c.big names it).
int tsvector_cast(const char *who, const TsvVocab &v, const uint8_t seed[32], const bm25x_tsvectors *t, int as_query,
                  TsvCast &c);
// Rows of a cast: row i = ord / tf [off[i], off[i+1]); len[i] = the saturating Σ tf of row i (document mode).
struct TsvRows {
    std::vector<uint64_t> off;
    std::vector<uint32_t> ord, tf, len;
};
// number(nu, keys, ord): ord[i] = the ordinal of keys[16 i .. 16 i + 16) (the keys ascending and distinct), or a refusal.
using TsvNumbering = std::function<int(uint32_t nu, const uint8_t *keys, uint32_t *ord)>;
// The cast of t (checked) on v.device with each key's ordinal in v's vocabulary.  Query mode: BM25X_TERM_MISSING where
// the vocabulary lacks the key.  Document mode: the keys it lacks go to `number` once each, and every row comes back
// ascending by ordinal with the tf of its merged counts; more than 2^31 - 1 elements or tsvectors is
// BM25X_ERR_UNSUPPORTED.  Refusals: the cast's, number's, CUDA failures named by who.
int tsvector_rows(const char *who, const TsvVocab &v, const uint8_t seed[32], const bm25x_tsvectors *t, int as_query,
                  const TsvNumbering &number, TsvRows &out);

// ---- host checks and helpers shared by the builders, with the messages their refusals give ----

int cuda_refusal(const char *who, const char *step, cudaError_t e);
int check_device(const char *who, int device);
int check_common(const char *who, uint32_t n_docs, const void *doc_len, double k1, double b, int device);
int check_keys(const char *who, const uint8_t *term_key, uint32_t T);
// address_tokens::read: the ordinal of the 16-byte key in the strictly ascending keys[0..T), or BM25X_TERM_MISSING.
uint32_t key_ordinal(const uint8_t *keys, uint32_t T, const uint8_t *key);
int check_shard_args(uint32_t N, uint32_t S, const uint32_t *doc_bounds);
std::vector<uint32_t> shard_bounds(const uint32_t *doc_bounds, const std::vector<uint64_t> &cum, uint32_t N,
                                   uint32_t S);
uint8_t bm25x_length_to_fieldnorm(uint32_t len);
uint64_t doc_norms(uint32_t N, const uint32_t *doc_len, const uint8_t *stored_fn, uint64_t stored_sum, uint8_t *fn);
void synth_ctid(uint32_t g, uint16_t *out);

// One sealed handle's documents: the handle, the id of its local document 0 in the whole segment, its documents.
struct SealPart {
    bm25x_index *h;
    uint32_t first, n;
};

// The sealed side of a growing segment or a search: one index (ix), or a document-sharded index (sx).  It answers for the
// whole segment (n_docs, n_terms, df, Σlen, avgdl, keys: shard 0 holds them) and names the handle the growing segment
// lives beside, `home`: the index, or the LAST shard (device, SM count, options), where the growing documents sit in id
// order.
struct SealedSide {
    bm25x_index *ix = nullptr;
    bm25x_sharded_index *sx = nullptr;

    const bm25x_index &home() const { return sx ? *sx->shards.back() : *ix; }
    uint32_t n_docs() const { return sx ? sx->n_docs : ix->d.n_docs; }
    uint32_t n_terms() const { return sx ? sx->n_terms : ix->d.n_terms; }
    const std::vector<uint32_t> &df() const { return sx ? sx->h_df : ix->h_df; }
    const std::vector<uint8_t> &keys() const { return sx ? sx->shards[0]->h_keys : ix->h_keys; }
    // the statistics of the whole sealed segment: the growing segment scores with them (search.rs:66-77), not its own
    Stats stats() const {
        const bm25x_index &h = home();
        return sx ? Stats(sx->n_docs, sx->sum_len, sx->avgdl, sx->h_df.data(), sx->n_terms, h.k1, h.b)
                  : Stats(ix->d.n_docs, ix->sum_len, ix->avgdl, ix->h_df.data(), ix->d.n_terms, h.k1, h.b);
    }
    std::vector<SealPart> parts() const {
        if (!sx) return {{ix, 0, ix->d.n_docs}};
        std::vector<SealPart> p;
        for (uint32_t s = 0; s < sx->n_shards; s++)
            p.push_back({sx->shards[s], sx->bounds[s], sx->bounds[s + 1] - sx->bounds[s]});
        return p;
    }
};

// What each list of a sealed-side search selects: prefilter bitmaps (allow_sealed over the side's global ids,
// allow_growing over the growing handle's ordinals; NULL = all pass), or, when c_off is set, candidate lists
// (bm25x_search_candidates) in the result id space: sealed ids, then growing ordinal o as n_docs() + o.
struct SideFilter {
    const uint8_t *allow_sealed = nullptr, *allow_growing = nullptr;
    const uint32_t *c_off = nullptr, *c_docs = nullptr;
};

// The search of a sealed side and, when `growing` is given, a growing handle over ids n_docs() + ordinal (bm25x_shards.cu).
// One index without a growing handle: bm25x_search_batch, or bm25x_search_candidates.  Otherwise every part's top-k and
// the growing handle's, merged on the device: with its slice of allow_sealed / with allow_growing, or with the candidates
// that fall in its id range, as local ids.  A sharded side first makes bm25x_search_batch's request checks and
// canonicalises the queries against the whole segment, so that its refusals are those of the unsharded index; candidates
// at or past the last id of the side and the growing handle are refused next.  stats->queries = the live queries of the
// whole sealed segment, plus the growing handle's when count_growing; h2d_ms is counted from t0.  CUDA failures and the
// candidates' refusals are named by `who`.
int sealed_side_search(const char *who, const SealedSide &sealed, bm25x_index *growing, const SideFilter &f,
                       bool count_growing, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms, uint32_t k,
                       const ResultRows &host, bm25x_search_stats *stats, std::chrono::steady_clock::time_point t0);

// The container of a document-sharded build, for every source: after the host checks of the segment c (P postings, df,
// the statistics st), every shard's device is checked with who's message; then prepare(device of shard 0, cum) runs the
// host work and refusals that need a device and, when doc_bounds is NULL, gives the postings per document for the balanced
// bounds (shard_bounds); then the shards are built one at a time by build(s, device, lo, hi, ix).  c->n_terms, P, df and
// st are read after prepare, which may set them.  On the first failure everything built so far is destroyed.
template <typename Segment, typename Prepare, typename Build>
int sharded_build(const char *who, const Segment *c, const uint64_t &P, const std::vector<uint32_t> &df, const Stats &st,
                  uint32_t S, const uint32_t *doc_bounds, const int *devices, Prepare prepare, Build build,
                  bm25x_sharded_index **out) {
    std::vector<int> dev(S, 0);
    if (devices) std::copy(devices, devices + S, dev.begin());
    for (uint32_t s = 0; s < S; s++) {
        const int rc = check_device(who, dev[s]);
        if (rc != BM25X_OK) return rc;
    }
    std::vector<uint64_t> cum;
    int rc = prepare(dev[0], doc_bounds ? nullptr : &cum);
    if (rc != BM25X_OK) return rc;
    std::unique_ptr<bm25x_sharded_index, void (*)(bm25x_sharded_index *)> sx(new bm25x_sharded_index(),
                                                                             bm25x_sharded_destroy);
    sx->n_shards = S;
    sx->bounds = shard_bounds(doc_bounds, cum, c->n_docs, S);
    std::vector<uint64_t>().swap(cum);
    sx->n_docs = c->n_docs;
    sx->n_terms = c->n_terms;
    sx->n_post = P;
    sx->k1 = c->k1;
    sx->b = c->b;
    sx->h_df = df;
    sx->sum_len = st.sum_len;
    sx->avgdl = st.avgdl;
    for (uint32_t s = 0; s < S; s++) {
        IndexGuard ix;
        rc = build(s, dev[s], sx->bounds[s], sx->bounds[s + 1], ix);
        if (rc != BM25X_OK) return rc;
        sx->shards.push_back(ix.release());
    }
    *out = sx.release();
    return BM25X_OK;
}
