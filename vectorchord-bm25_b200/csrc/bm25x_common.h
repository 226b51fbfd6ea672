// bm25x_common.h — internal types shared by the host library and the sm_90a kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <array>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/bm25x.h"

#define BM25X_BLOCK 128u            // postings per block, as the reference (crates/bm25/src/flush.rs:84)
#define BM25X_DOC_INF 0xFFFFFFFFu   // exhausted-cursor sentinel, as search.rs:484-496
#define BM25X_POST_ALIGN 4u         // every term's posting list starts on a multiple of 4 postings: 16-byte TMA granularity of
                                    // the doc-id-only copy (pdoc, 4 B per posting) as well as of the 8-byte postings
#define BM25X_CHAMP_L 128u          // champion list: the best min(df, 128) postings of every term by single-term score
#define BM25X_POST_SLACK 4u         // slack slots behind the last list, reading as exhausted cursors

// The five launch flavours of the search kernel k_search_ring (bm25x_search_ring.cuh, RCfg::FLAVOUR).
enum RingFlavour : int {
    RING_PLAIN = 0,     // one launch answers its queries (8-byte postings in the rings, MaxScore pruning)
    RING_SUSPEND = 1,   // two-phase launches, first: the plain kernel, which suspends a query once no posting can pass alone
    RING_RESUME = 2,    // two-phase launches, second: doc-id-only rings resume the suspended queries
    RING_SEEDED = 3,    // single-term documents from the champion lists, doc-id-only rings, no pruning
    RING_HANDBACK = 4,  // the plain kernel over the queries a seeded launch handed back
};

void bm25x_set_error(const char *fmt, ...);
// Host threads this process may really use: the affinity mask capped by the cgroup CPU quota (omp_get_max_threads()
// ignores the quota: 128 threads spinning on a dozen granted cores cost the batch canonicalisation tens of ms).
int bm25x_host_threads(int cap);

#define BM25X_CUDA_TRY(expr)                                                                   \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            bm25x_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,  \
                            __LINE__);                                                         \
            return _e == cudaErrorMemoryAllocation ? BM25X_ERR_OOM : BM25X_ERR_CUDA;           \
        }                                                                                      \
    } while (0)

// A posting as it lives in HBM: 8 bytes, the reference's logical Mapping(doc u32, tf u32)
// (segment.rs:23-25) with the document's fieldnorm byte folded into the low 8 bits of the
// second word: w = tf << 8 | fieldnorm(doc).  tf < 2^24 is enforced at index build.
struct Posting {
    uint32_t doc;
    uint32_t w;
};

// Device-resident index (flat arrays; replaces the reference's 8 KiB pages, tapes and address trees).
struct DeviceIndex {
    uint32_t n_docs = 0, n_terms = 0;
    uint64_t n_post = 0;      // real postings
    uint64_t n_post_pad = 0;  // incl. the pad slots that round every term up to BM25X_POST_ALIGN postings
    uint64_t n_blocks = 0;
    Posting *post = nullptr;        // [n_post_pad] term-major, doc-ascending inside a term
    uint32_t *pdoc = nullptr;       // [n_post_pad] the doc ids of `post` alone (derived on the device, not replicated): what the
                                    // 2..4-term classes of k_search_ring stream — their hot loop never reads tf / fieldnorm
    // Champion lists (derived on the device, not replicated): per term its best min(df, BM25X_CHAMP_L) postings in the
    // result order (exact single-term score desc, doc id asc).  A document that holds ONE query term can only be in the
    // top-k if it is among the first k champions of that term (every posting ranked before it belongs to a document that
    // beats it), so a query seeds its pool from these and its stream never tests single postings (RCfg::SEEDED).
    Posting *champ = nullptr;       // [champ_off[n_terms]]
    uint64_t *champ_off = nullptr;  // [n_terms+1]
    uint64_t n_champ = 0;
    uint64_t *post_off = nullptr;   // [n_terms+1] padded offsets (multiples of BM25X_POST_ALIGN)
    uint32_t *df = nullptr;         // [n_terms] TokenTuple.number_of_documents
    uint64_t *blk_off = nullptr;    // [n_terms+1] first block index of each term
    uint2 *blk = nullptr;           // [n_blocks] (first doc, last doc) — SummaryTuple.{min,max}_document_id
    float *blk_ub = nullptr;        // [n_blocks] upper bound of one posting's score inside the block (SummaryTuple.wand_*)
    float *s0f = nullptr;           // [n_terms] float(s0)
    double *s0d = nullptr;          // [n_terms] idf*(k1+1), bm25.rs:348
    double *s1d = nullptr;          // [256] k1*(1-b+b*len(fn)/avgdl), bm25.rs:349-352
    float *s1f = nullptr;           // [256]
    double *ubd = nullptr;          // [n_terms] upper bound of one posting's exact score (token-level WAND bound)
    uint8_t *fieldnorm = nullptr;   // [n_docs]
    uint16_t *payload = nullptr;    // [n_docs*3]
};

struct bm25x_index {
    int device = 0;
    int sm_count = 0;
    DeviceIndex d;
    double k1 = 1.2, b = 0.75, avgdl = 0;
    float s1f_min = 0.f;               // min over the documents of s1f[fieldnorm]: one-compare single-term test (k_search_ring)
    uint64_t sum_len = 0;
    uint64_t device_bytes = 0;
    std::vector<uint32_t> h_df;        // host copy for query canonicalisation
    std::vector<uint8_t> h_keys;       // [n_terms*16] sorted keys (optional)
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;  // bm25x_search_batch: result downloads of one slice while the next one runs
    uint32_t slice_min = 32768;          // bm25x_search_batch cuts batches of >= 2 x this many queries into slices (0: never)
    std::vector<void *> allocs;
    int prune = 1;                     // MaxScore-style pruning in the search kernels
    uint32_t seed_dense_div = 64;      // seeded launches hand queries with a list of n_docs / 64 postings or more to the plain kernel
    uint32_t seed_prune_min = 32768;   // seeded launches hand queries with a list this long (and 8x their shortest) to the pruning kernel
    int seed_max_terms = 8;            // widest term-count class that runs seeded (4 or 8)
    int seed = 1;                      // 2..4-term classes, k <= BM25X_CHAMP_L, no prefilter: pools seeded from the champion lists
    int twophase = 0;                  // 2..4-term classes, k <= 224: two launches (8-byte postings, then doc ids only)
    // page-locked staging buffer of bm25x_batch_prepare (grow-only, shared by the batches of this index)
    uint32_t *h_stage = nullptr;
    size_t h_stage_words = 0;
    cudaEvent_t h_stage_free = nullptr;  // recorded after the upload that last read h_stage
    bool h_stage_busy = false;
    std::mutex stage_mutex;
    // bm25x_evaluate_batch: tables that depend on the index alone, built on first use (idf per term with the host libm,
    // fieldnorm -> length), kept on the device
    double *eval_idf = nullptr;
    uint32_t *eval_fn_len = nullptr;
    std::mutex eval_mutex;
};

// Document-sharded index (bm25x_sharded_*): shard s is an ordinary index over the documents [bounds[s], bounds[s+1]) with
// local ids, built with the whole segment's statistics (one Stats object), so it scores with the same s0 / s1 bits.
struct bm25x_sharded_index {
    uint32_t n_shards = 0;
    std::vector<uint32_t> bounds;        // [n_shards+1]
    std::vector<bm25x_index *> shards;   // [n_shards]
    // the whole segment, as bm25x_index_get_info / query canonicalisation see it
    uint32_t n_docs = 0, n_terms = 0;
    uint64_t n_post = 0, sum_len = 0;
    double k1 = 1.2, b = 0.75, avgdl = 0;
    std::vector<uint32_t> h_df;
};

// ---- internal to the host library (bm25x_search.cu, bm25x_shards.cu) ----

// Canonical queries (sort + dedup: datatype/tsvector.rs:96-105; unknown and df-0 terms dropped: search.rs:55-62).  Query i
// of q_off[0..nq] (absolute offsets into q_terms: q_off may be a slice of a longer array) keeps its live terms in place of
// its raw ones, at terms[q_off[i] - q_off[0]]; a query of 33..64 live terms holds its 32 rarest first, both groups
// ascending.  Refuses offsets that go backwards and more than BM25X_MAX_QUERY_TERMS live terms with the messages of
// bm25x_batch_prepare, naming the highest-numbered offending query of the slice.
struct CanonQueries {
    std::unique_ptr<uint32_t[]> terms;
    std::unique_ptr<uint32_t[]> live;  // live terms per query
    std::unique_ptr<uint64_t[]> cost;  // Σ df per query
};
int bm25x_canonicalise(const uint32_t *h_df, uint32_t n_terms, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                       CanonQueries *out);

// The slices bm25x_search_batch cuts a batch of nq queries into: min(16, nq / slice_min) of them when nq >= 2 x slice_min
// (slice_min != 0), else one.  Slice s holds the queries [begin(s), begin(s + 1)).
struct SlicePlan {
    uint32_t nq, n;
    SlicePlan(uint32_t slice_min, uint32_t nq_)
        : nq(nq_), n(slice_min && nq_ >= 2ull * slice_min ? std::min<uint32_t>(16u, nq_ / slice_min) : 1u) {}
    uint32_t begin(uint32_t s) const { return (uint32_t)(((uint64_t)nq * s) / n); }
};

// Result rows of a batch: per query k slots of doc id, f32 score, f64 score and payload (3 x u16), and the count n of
// filled slots.  An empty slot is doc BM25X_DOC_INF with zeros elsewhere.  Pointers are device or host memory.
struct ResultRows {
    uint32_t *doc = nullptr;
    float *score = nullptr;
    double *score64 = nullptr;
    uint16_t *payload = nullptr;
    uint32_t *n = nullptr;

    // bytes of the five arrays for `rows` queries
    static std::array<size_t, 5> bytes(size_t rows, uint32_t k) {
        const size_t slots = rows * k;
        return {4 * slots, 4 * slots, 8 * slots, 6 * slots, 4 * rows};
    }
    std::array<void *, 5> arrays() const { return {doc, score, score64, payload, n}; }
    // the rows from query `row` on (null arrays stay null)
    ResultRows from(size_t row, uint32_t k) const {
        ResultRows r;
        if (doc) r.doc = doc + row * k;
        if (score) r.score = score + row * k;
        if (score64) r.score64 = score64 + row * k;
        if (payload) r.payload = payload + row * k * 3;
        if (n) r.n = n + row;
        return r;
    }
    // stream-ordered device memory for `rows` queries
    cudaError_t alloc(size_t rows, uint32_t k, cudaStream_t st) {
        void **p[5] = {(void **)&doc, (void **)&score, (void **)&score64, (void **)&payload, (void **)&n};
        const auto b = bytes(rows, k);
        cudaError_t e = cudaSuccess;
        for (int a = 0; a < 5 && e == cudaSuccess; a++) e = cudaMallocAsync(p[a], b[a] ? b[a] : 8, st);
        return e;
    }
    void release(cudaStream_t st) {
        for (void *p : arrays())
            if (p) cudaFreeAsync(p, st);
        *this = ResultRows();
    }
    // every slot empty, every count 0
    cudaError_t reset(size_t rows, uint32_t k, cudaStream_t st) const {
        const auto p = arrays();
        const auto b = bytes(rows, k);
        cudaError_t e = cudaSuccess;
        for (int a = 0; a < 5 && e == cudaSuccess; a++) e = cudaMemsetAsync(p[a], a == 0 ? 0xFF : 0, b[a], st);
        return e;
    }
    // the first `rows` queries into dst (host memory or another device's: the copy kind follows the addresses), skipping
    // the arrays dst leaves null
    cudaError_t copy_to(const ResultRows &dst, size_t rows, uint32_t k, cudaStream_t st) const {
        const auto s = arrays(), d = dst.arrays();
        const auto b = bytes(rows, k);
        cudaError_t e = cudaSuccess;
        for (int a = 0; a < 5 && e == cudaSuccess; a++)
            if (d[a] && b[a]) e = cudaMemcpyAsync(d[a], s[a], b[a], cudaMemcpyDefault, st);
        return e;
    }
};

// A prepared batch (bm25x_batch_prepare) seen from the sharded search: its output rows; a run on its index's stream between
// the batch's timing events, without synchronising; the event that closes that run; after it has finished, its figures
// added to *acc.
const ResultRows &bm25x_batch_rows(const bm25x_batch *b);
int bm25x_batch_run_timed(bm25x_batch *b);
cudaEvent_t bm25x_batch_done_event(bm25x_batch *b);
int bm25x_batch_add_stats(bm25x_batch *b, bm25x_search_stats *acc);
