// bm25x_search.cu — batched BM25 top-k over the HBM-resident index (sm_90a).
//
// Replaces bm25::search (crates/bm25/src/search.rs:28-282): instead of one query walking cursors
// over 8 KiB pages with Block-max WAND, a persistent grid streams every query's posting lists
// through shared memory with TMA bulk copies and merges them there.
//
//   k_search_ring (bm25x_search_ring.cuh): one warp per query, persistent grid.  Every term owns a shared-memory ring
//   filled by TMA bulk copies; the runs of a doc window are united through a presence map (test against the marks of
//   the earlier runs, then mark), detected postings are verified by binary search, filtered in f32 and re-scored in
//   f64 in the reference's operation order; MaxScore pruning with probes of the pruned terms in HBM.
//
// Exactness: the f32 filter only ever *rejects* documents whose f32 score is below Sk·(1-2^-18) where Sk is the
// exact f64 k-th best so far; the f32 error bound is < 2^-18 relative (DESIGN.md §5); everything that survives is
// ranked by its exact f64 score.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <mutex>
#include <vector>

#include "bm25x_build.h"

#include "bm25x_device.cuh"

// =============================================================================================
// Host side
// =============================================================================================

static const int kClasses[] = {1, 2, 3, 4, 8, 16, 32, 64};  // 64: two passes of the 32-term kernel (33..64 live terms)
static const int kNumClasses = 8;

struct Group {
    int M = 0;
    uint32_t nq = 0;
    uint32_t *d_ids = nullptr, *d_off = nullptr, *d_terms = nullptr;  // slices of one device buffer
    int *d_counter = nullptr;
    // two-phase launches (2..4 terms, k <= 224): suspended-query list + hand-over records (bm25x_device.cuh)
    uint32_t *d_q2 = nullptr;
    ResumeRec *d_resume = nullptr;
};

struct bm25x_batch {
    bm25x_index *ix = nullptr;
    uint32_t nq = 0, k = 0;
    Group groups[kNumClasses];
    uint8_t *d_allow = nullptr;
    ResultRows out;  // [nq] rows of k slots on the device
    unsigned long long *d_fetched = nullptr;
    uint64_t postings = 0, qterms = 0;
    uint32_t live = 0;
    uint32_t launches = 0;  // issued by the last run
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_ready = nullptr;
    std::vector<void *> allocs;
    void *last_stream = nullptr;
};

// kernel v6 (bm25x_search_ring.cu: warp per query, ring stages + presence map), one entry per pool capacity
// flavour: which launch of the class this is (RingFlavour, bm25x_common.h)
int bm25x_launch_ring_kp64(int device, int sm_count, const SearchParams &sp, int M, RingFlavour flavour, cudaStream_t stream);
int bm25x_launch_ring_kp256(int device, int sm_count, const SearchParams &sp, int M, RingFlavour flavour, cudaStream_t stream);
int bm25x_launch_ring_kp2048(int device, int sm_count, const SearchParams &sp, int M, RingFlavour flavour, cudaStream_t stream);
int bm25x_launch_ring_kp131072(int device, int sm_count, const SearchParams &sp, int M, RingFlavour flavour, cudaStream_t stream);

// Two launches per class: 2..4 terms with the pool in shared memory (k <= 224).
static bool two_phase_class(const bm25x_index *ix, int M, uint32_t k) { return ix->twophase && M >= 2 && M <= 4 && k <= 224; }
// One seeded launch (RING_SEEDED): 2..4 terms, k within the champion lists, no prefilter bitmap (a filtered-out champion would
// have to be replaced by the next one of its term: such batches take the unseeded kernels).
static bool seeded_class(const bm25x_index *ix, int M, uint32_t k, const uint8_t *allow) {
    return ix->seed && ix->d.champ && !allow && M >= 2 && M <= ix->seed_max_terms && k <= BM25X_CHAMP_L;
}

static int launch_ring_k(const bm25x_index *ix, const SearchParams &sp, int M, RingFlavour flavour, cudaStream_t stream) {
    if (sp.k <= 32) return bm25x_launch_ring_kp64(ix->device, ix->sm_count, sp, M, flavour, stream);
    if (sp.k <= 224) return bm25x_launch_ring_kp256(ix->device, ix->sm_count, sp, M, flavour, stream);
    if (sp.k <= 1024) return bm25x_launch_ring_kp2048(ix->device, ix->sm_count, sp, M, RING_PLAIN, stream);
    return bm25x_launch_ring_kp131072(ix->device, ix->sm_count, sp, M, RING_PLAIN, stream);  // candidate pools in HBM
}

template <typename T>
static int batch_alloc(bm25x_batch *b, T **p, size_t n) {
    // stream-ordered allocation from the device's (cached) default pool: no cudaMalloc/cudaFree cost per call
    BM25X_CUDA_TRY(cudaMallocAsync((void **)p, sizeof(T) * (n ? n : 1), b->ix->stream));
    b->allocs.push_back((void *)*p);
    return BM25X_OK;
}

extern "C" void bm25x_batch_destroy(bm25x_batch *b) {
    if (!b) return;
    cudaSetDevice(b->ix->device);
    if (b->last_stream && b->last_stream != (void *)b->ix->stream) cudaStreamSynchronize((cudaStream_t)b->last_stream);
    for (void *p : b->allocs) cudaFreeAsync(p, b->ix->stream);
    b->out.release(b->ix->stream);
    if (b->ev0) cudaEventDestroy(b->ev0);
    if (b->ev1) cudaEventDestroy(b->ev1);
    if (b->ev_ready) cudaEventDestroy(b->ev_ready);
    delete b;
}

#define BTRY(x)                      \
    do {                             \
        int _rc = (x);               \
        if (_rc != BM25X_OK) {       \
            bm25x_batch_destroy(b);  \
            return _rc;              \
        }                            \
    } while (0)

// OpenMP over the queries; no per-query allocation.
int bm25x_canonicalise(const uint32_t *h_df, uint32_t n_terms, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                       CanonQueries *out) {
    const size_t base0 = nq ? q_off[0] : 0;
    const size_t n_raw = nq && q_off[nq] >= base0 ? q_off[nq] - base0 : 0;
    // not zeroed: the loop writes every query's entries (the first touch of the pages is spread over the threads)
    out->terms.reset(new uint32_t[n_raw ? n_raw : 1]);
    out->live.reset(new uint32_t[nq ? nq : 1]);
    out->cost.reset(new uint64_t[nq ? nq : 1]);
    uint32_t *const canon = out->terms.get(), *const live = out->live.get();
    uint64_t *const cost = out->cost.get();
    int bad = -1;  // the highest-numbered offending query, whatever the thread count
    const int nthr = nq < 4096 ? 1 : bm25x_host_threads(16);  // small batches: a parallel region costs more than the loop
#pragma omp parallel for schedule(static, 1024) num_threads(nthr) reduction(max : bad)
    for (uint32_t i = 0; i < nq; ++i) {
        if (q_off[i + 1] < q_off[i] || q_off[i] < base0 || q_off[i + 1] - base0 > n_raw) {
            bad = std::max(bad, (int)i);
            live[i] = 0;
            cost[i] = 0;
            continue;
        }
        uint32_t *dst = canon + (q_off[i] - base0);
        const uint32_t n = q_off[i + 1] - q_off[i];
        uint32_t m = 0;
        for (uint32_t j = 0; j < n; ++j) {
            const uint32_t t = q_terms[q_off[i] + j];
            if (t < n_terms && h_df[t] != 0) dst[m++] = t;
        }
        std::sort(dst, dst + m);
        m = (uint32_t)(std::unique(dst, dst + m) - dst);
        uint64_t cst = 0;
        for (uint32_t j = 0; j < m; ++j) cst += h_df[dst[j]];
        cost[i] = cst;
        if (m > 32 && m <= BM25X_MAX_QUERY_TERMS) {
            // two-pass query: the 32 rarest terms first (group 0, streamed by the first pass), the others after them;
            // both groups ascending — the kernel merges them back into ascending term order for the exact sum
            uint32_t tmp[BM25X_MAX_QUERY_TERMS];
            std::copy(dst, dst + m, tmp);
            std::nth_element(tmp, tmp + 32, tmp + m, [&](uint32_t a, uint32_t b) {
                return h_df[a] != h_df[b] ? h_df[a] < h_df[b] : a < b;
            });
            std::sort(tmp, tmp + 32);
            std::sort(tmp + 32, tmp + m);
            std::copy(tmp, tmp + m, dst);
        }
        if (m > BM25X_MAX_QUERY_TERMS) bad = std::max(bad, (int)i);
        live[i] = m;
    }
    if (bad < 0) return BM25X_OK;
    if (live[bad] == 0) {  // offsets (a query with too many live terms has more than 0)
        bm25x_set_error("bm25x_batch_prepare: q_off not monotone at %d", bad);
        return BM25X_ERR_INVALID;
    }
    bm25x_set_error("bm25x_batch_prepare: query %d has %u live terms > %d", bad, live[bad], BM25X_MAX_QUERY_TERMS);
    return BM25X_ERR_UNSUPPORTED;
}

int check_queries(uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms) {
    if (nq && (!q_off || (!q_terms && q_off[nq] != 0))) {
        bm25x_set_error("bm25x_batch_prepare: null argument");
        return BM25X_ERR_INVALID;
    }
    return BM25X_OK;
}

int check_k(uint32_t k, bool max_k) {
    if (k == 0) {
        bm25x_set_error("number of needed rows is set to 0");  // scanners/default.rs:114-116
        return BM25X_ERR_LIMIT_ZERO;
    }
    if (max_k && k > BM25X_MAX_K) {
        bm25x_set_error("bm25x_batch_prepare: k=%u > BM25X_MAX_K=%d", k, BM25X_MAX_K);
        return BM25X_ERR_UNSUPPORTED;
    }
    return BM25X_OK;
}

int stage_reserve(bm25x_index *ix, const char *who, size_t words, uint32_t **out) {
    if (ix->h_stage_words < words) {
        if (ix->h_stage) {
            cudaStreamSynchronize(ix->stream);  // an earlier batch's upload may still read it
            cudaFreeHost(ix->h_stage);
        }
        ix->h_stage = nullptr;
        ix->h_stage_words = 0;
        const size_t cap = words + words / 4 + 1024;
        const cudaError_t e = cudaMallocHost((void **)&ix->h_stage, cap * sizeof(uint32_t));
        if (e != cudaSuccess) {
            bm25x_set_error("%s: page-locked staging buffer: %s", who, cudaGetErrorString(e));
            return BM25X_ERR_OOM;
        }
        ix->h_stage_words = cap;
    } else if (ix->h_stage_busy) {
        cudaEventSynchronize(ix->h_stage_free);  // the previous upload from this buffer has been issued; wait for it
    }
    *out = ix->h_stage;
    return BM25X_OK;
}

cudaError_t stage_upload(bm25x_index *ix, void *d, size_t words) {
    cudaError_t e = cudaMemcpyAsync(d, ix->h_stage, words * sizeof(uint32_t), cudaMemcpyHostToDevice, ix->stream);
    if (e == cudaSuccess) {
        if (!ix->h_stage_free) e = cudaEventCreateWithFlags(&ix->h_stage_free, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventRecord(ix->h_stage_free, ix->stream);
        ix->h_stage_busy = true;
    }
    return e;
}

// Canonicalises the queries (bm25x_canonicalise), groups them by term-count class and uploads everything with ONE copy
// from a page-locked staging buffer cached in the index handle.
extern "C" int bm25x_batch_prepare(bm25x_index *ix, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                                   uint32_t k, const uint8_t *allow, bm25x_batch **out) {
    if (!ix || !out) {
        bm25x_set_error("bm25x_batch_prepare: null argument");
        return BM25X_ERR_INVALID;
    }
    if (const int rc = check_queries(nq, q_off, q_terms); rc != BM25X_OK) return rc;
    *out = nullptr;
    if (ix->h_df.size() != ix->d.n_terms) {
        bm25x_set_error("bm25x_batch_prepare: replica not finalized (bm25x_index_finalize_replica)");
        return BM25X_ERR_INVALID;
    }
    if (const int rc = check_k(k, true); rc != BM25X_OK) return rc;
    const uint32_t *h_df = ix->h_df.data();
    CanonQueries cq;
    const int crc = bm25x_canonicalise(h_df, ix->d.n_terms, nq, q_off, q_terms, &cq);
    if (crc != BM25X_OK) return crc;
    const size_t base0 = nq ? q_off[0] : 0;
    const uint32_t *const canon = cq.terms.get(), *const live = cq.live.get();
    const uint64_t *const cost = cq.cost.get();
    const int nthr = nq < 4096 ? 1 : bm25x_host_threads(16);
    bm25x_batch *b = new bm25x_batch();
    b->ix = ix;
    b->nq = nq;
    b->k = k;
    uint64_t b_qterms = 0;
    uint32_t b_live = 0;
    // ---- slots: inside a class the queries are ordered HEAVIEST FIRST (Σ df in power-of-two buckets): the persistent
    // kernels hand queries out in slot order, so the long head-term queries start first and the tail of the launch is made
    // of short ones (longest-processing-time scheduling; matters for skewed term frequencies, BASELINE configs[3]).
    // query i is the slot[i]-th query of its class, its terms start at tpos[i] inside the class ----
    uint8_t cls_of[BM25X_MAX_QUERY_TERMS + 1];
    for (int m = 0, c = 0; m <= BM25X_MAX_QUERY_TERMS; ++m) {
        while (kClasses[c] < m) ++c;
        cls_of[m] = (uint8_t)c;
    }
    constexpr int NB = 48;  // cost buckets per class
    std::vector<uint32_t> slot(nq ? nq : 1), tpos(nq ? nq : 1);
    std::vector<uint8_t> bucket(nq ? nq : 1);
    static_assert(kNumClasses * NB <= 512, "bucket table");
    uint32_t bq[kNumClasses * NB] = {0}, bt[kNumClasses * NB] = {0};
    for (uint32_t i = 0; i < nq; ++i) {
        const uint32_t m = live[i];
        if (!m) continue;
        const int c = cls_of[m];
        const int b = NB - 1 - std::min<int>(NB - 1, 63 - __builtin_clzll(cost[i] | 1ull));  // 0 = heaviest
        bucket[i] = (uint8_t)b;
        bq[c * NB + b]++;
        bt[c * NB + b] += m;
        b_qterms += m;
        b_live++;
    }
    uint32_t cnt_q[kNumClasses] = {0}, cnt_t[kNumClasses] = {0};
    for (int c = 0; c < kNumClasses; ++c) {
        uint32_t q0 = 0, t0 = 0;
        for (int b = 0; b < NB; ++b) {  // exclusive prefix inside the class
            const uint32_t nqb = bq[c * NB + b], ntb = bt[c * NB + b];
            bq[c * NB + b] = q0;
            bt[c * NB + b] = t0;
            q0 += nqb;
            t0 += ntb;
        }
        cnt_q[c] = q0;
        cnt_t[c] = t0;
    }
    for (uint32_t i = 0; i < nq; ++i) {
        const uint32_t m = live[i];
        if (!m) continue;
        const int key = cls_of[m] * NB + bucket[i];
        slot[i] = bq[key]++;
        tpos[i] = bt[key];
        bt[key] += m;
    }
    b->qterms = b_qterms;
    b->live = b_live;
    // one staging / device buffer: per class [ids | off | terms | work counter]
    size_t base_ids[kNumClasses], base_off[kNumClasses], base_terms[kNumClasses], base_cnt[kNumClasses], words = 0;
    for (int c = 0; c < kNumClasses; ++c) {
        Group &g = b->groups[c];
        g.M = kClasses[c];
        g.nq = cnt_q[c];
        base_ids[c] = words;
        words += cnt_q[c];
        base_off[c] = words;
        words += (size_t)cnt_q[c] + 1;
        base_terms[c] = words;
        words += cnt_t[c];
        base_cnt[c] = words;
        words += 1;
    }
    cudaError_t e = cudaSetDevice(ix->device);
    if (e != cudaSuccess) {
        bm25x_set_error("cudaSetDevice: %s", cudaGetErrorString(e));
        delete b;
        return BM25X_ERR_CUDA;
    }
    cudaStream_t st = ix->stream;
    std::lock_guard<std::mutex> stage_lock(ix->stage_mutex);  // the staging buffer is shared by the batches of this index
    uint32_t *hs = nullptr;
    if (const int rc = stage_reserve(ix, "bm25x_batch_prepare", words, &hs); rc != BM25X_OK) {
        delete b;
        return rc;
    }
    for (int c = 0; c < kNumClasses; ++c) {
        hs[base_off[c]] = 0;
        hs[base_cnt[c]] = 0;
    }
    uint64_t postings = 0;
    // ---- pass 2 (parallel): scatter into the staging buffer ----
#pragma omp parallel for schedule(static, 1024) reduction(+ : postings) num_threads(nthr)
    for (uint32_t i = 0; i < nq; ++i) {
        const uint32_t m = live[i];
        if (!m) continue;
        const int c = cls_of[m];
        hs[base_ids[c] + slot[i]] = i;
        hs[base_off[c] + slot[i] + 1] = tpos[i] + m;
        const uint32_t *src = canon + (q_off[i] - base0);
        uint32_t *dst = hs + base_terms[c] + tpos[i];
        for (uint32_t j = 0; j < m; ++j) {
            dst[j] = src[j];
            postings += h_df[src[j]];
        }
    }
    b->postings = postings;
    uint32_t *d_q = nullptr;
    BTRY(batch_alloc(b, &d_q, words));
    e = stage_upload(ix, d_q, words);
    for (int c = 0; c < kNumClasses; ++c) {
        Group &g = b->groups[c];
        g.d_ids = d_q + base_ids[c];
        g.d_off = d_q + base_off[c];
        g.d_terms = d_q + base_terms[c];
        g.d_counter = (int *)(d_q + base_cnt[c]);
    }
    if (allow && e == cudaSuccess) {
        size_t nb = ((size_t)ix->d.n_docs + 7) / 8;
        BTRY(batch_alloc(b, &b->d_allow, nb));
        e = cudaMemcpyAsync(b->d_allow, allow, nb, cudaMemcpyHostToDevice, st);
    }
    for (int c = 0; c < kNumClasses; ++c) {
        Group &g = b->groups[c];
        if (g.nq && (two_phase_class(ix, g.M, k) || seeded_class(ix, g.M, k, allow))) {
            BTRY(batch_alloc(b, &g.d_q2, (size_t)g.nq + 2));  // hand-over list of the class (suspended / handed-back queries)
            if (two_phase_class(ix, g.M, k)) BTRY(batch_alloc(b, &g.d_resume, (size_t)g.nq));
        }
    }
    BTRY(batch_alloc(b, &b->d_fetched, 1));
    if (e == cudaSuccess) e = b->out.alloc(nq, k, st);
    if (e == cudaSuccess) e = b->out.reset(nq, k, st);  // rows of queries without a live term are never written by a kernel
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev1);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&b->ev_ready, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(b->ev_ready, st);  // bm25x_batch_run on another stream waits for the upload
    if (e != cudaSuccess) {
        bm25x_set_error("bm25x_batch_prepare: %s", cudaGetErrorString(e));
        bm25x_batch_destroy(b);
        return e == cudaErrorMemoryAllocation ? BM25X_ERR_OOM : BM25X_ERR_CUDA;
    }
    *out = b;
    return BM25X_OK;
}

// The fields of the search kernels' parameters that depend on the index handle alone: its device arrays and options.
SearchParams index_params(const bm25x_index *ix) {
    const DeviceIndex &d = ix->d;
    SearchParams sp;
    sp.post = d.post;
    sp.pdoc = d.pdoc;
    sp.champ = d.champ;
    sp.champ_off = d.champ_off;
    sp.seed_prune_min = ix->seed_prune_min;
    sp.seed_dense_div = ix->seed_dense_div;
    sp.post_off = d.post_off;
    sp.df = d.df;
    sp.blk_off = d.blk_off;
    sp.blk = d.blk;
    sp.blk_ub = d.blk_ub;
    sp.s0f = d.s0f;
    sp.s0d = d.s0d;
    sp.s1d = d.s1d;
    sp.s1f = d.s1f;
    sp.payload = d.payload;
    sp.ubd = d.ubd;
    sp.prune = ix->prune;
    sp.s1f_min = ix->s1f_min;
    sp.n_docs = d.n_docs;
    return sp;
}

// The launches of one run on st, counted in b->launches.  Timed: the fetched-postings counter is zeroed and the run sits
// between the batch's events ev0 and ev1.  Does not synchronise.
static int batch_enqueue(bm25x_batch *b, cudaStream_t st, bool timed) {
    bm25x_index *ix = b->ix;
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    b->last_stream = (void *)st;
    if (st != ix->stream) BM25X_CUDA_TRY(cudaStreamWaitEvent(st, b->ev_ready, 0));  // uploads were issued on the library's stream
    uint32_t launches = 0;
    if (timed) {
        BM25X_CUDA_TRY(cudaMemsetAsync(b->d_fetched, 0, sizeof(unsigned long long), st));
        BM25X_CUDA_TRY(cudaEventRecord(b->ev0, st));
    }
    SearchParams sp = index_params(ix);
    sp.fetched = b->d_fetched;
    sp.k = b->k;
    sp.allow = b->d_allow;
    sp.out_doc = b->out.doc;
    sp.out_score = b->out.score;
    sp.out_score64 = b->out.score64;
    sp.out_payload = b->out.payload;
    sp.out_n = b->out.n;
    for (int c = 0; c < kNumClasses; ++c) {
        Group &g = b->groups[c];
        if (!g.nq) continue;
        sp.q_ids = g.d_ids;
        sp.q_off = g.d_off;
        sp.q_terms = g.d_terms;
        sp.nq = g.nq;
        sp.work_counter = g.d_counter;
        sp.q2 = g.d_q2;
        sp.resume = g.d_resume;
        BM25X_CUDA_TRY(cudaMemsetAsync(g.d_counter, 0, sizeof(int), st));
        int rc = BM25X_OK;
        if (g.d_q2 && seeded_class(ix, g.M, b->k, b->d_allow)) {
            // seeded launch (champion lists + doc-id-only stream, no pruning); the queries it hands back (a list much
            // longer than another: pruning pays) go through the plain kernel
            BM25X_CUDA_TRY(cudaMemsetAsync(g.d_q2, 0, 2 * sizeof(uint32_t), st));
            rc = launch_ring_k(ix, sp, g.M, RING_SEEDED, st);
            if (rc != BM25X_OK) return rc;
            launches++;
            rc = launch_ring_k(ix, sp, g.M, RING_HANDBACK, st);
        } else if (g.d_q2 && g.d_resume && ix->twophase) {
            // first phase: 8-byte postings until no posting can enter the top-k alone; second phase: the suspended
            // queries go on with doc ids only (bm25x_search_ring.cuh, RING_SUSPEND / RING_RESUME)
            BM25X_CUDA_TRY(cudaMemsetAsync(g.d_q2, 0, 2 * sizeof(uint32_t), st));
            rc = launch_ring_k(ix, sp, g.M, RING_SUSPEND, st);
            if (rc != BM25X_OK) return rc;
            launches++;
            rc = launch_ring_k(ix, sp, g.M, RING_RESUME, st);
        } else {
            rc = launch_ring_k(ix, sp, g.M, RING_PLAIN, st);
        }
        if (rc != BM25X_OK) return rc;
        launches++;
    }
    b->launches = launches;
    if (timed) BM25X_CUDA_TRY(cudaEventRecord(b->ev1, st));
    return BM25X_OK;
}

static int bm25x_batch_add_stats(bm25x_batch *b, bm25x_search_stats *acc);

extern "C" int bm25x_batch_run(bm25x_batch *b, void *stream_v, bm25x_search_stats *stats) {
    if (!b) {
        bm25x_set_error("bm25x_batch_run: null batch");
        return BM25X_ERR_INVALID;
    }
    const int rc = batch_enqueue(b, stream_v ? (cudaStream_t)stream_v : b->ix->stream, stats != nullptr);
    if (rc != BM25X_OK || !stats) return rc;
    BM25X_CUDA_TRY(cudaEventSynchronize(b->ev1));
    memset(stats, 0, sizeof(*stats));
    return bm25x_batch_add_stats(b, stats);
}

extern "C" int bm25x_batch_fetch(bm25x_batch *b, uint32_t *out_doc, float *out_score, double *out_score64,
                                 uint16_t *out_payload, uint32_t *out_n) {
    if (!b) {
        bm25x_set_error("bm25x_batch_fetch: null batch");
        return BM25X_ERR_INVALID;
    }
    BM25X_CUDA_TRY(cudaSetDevice(b->ix->device));
    cudaStream_t st = b->last_stream ? (cudaStream_t)b->last_stream : b->ix->stream;
    const ResultRows host{out_doc, out_score, out_score64, out_payload, out_n};
    BM25X_CUDA_TRY(b->out.copy_to(host, b->nq, b->k, st));
    BM25X_CUDA_TRY(cudaStreamSynchronize(st));
    return BM25X_OK;
}

extern "C" int bm25x_batch_device_results(bm25x_batch *b, void **doc, void **score, void **score64, void **payload,
                                          void **n) {
    if (!b) {
        bm25x_set_error("bm25x_batch_device_results: null batch");
        return BM25X_ERR_INVALID;
    }
    void **dst[5] = {doc, score, score64, payload, n};
    const auto p = b->out.arrays();
    for (int a = 0; a < 5; a++)
        if (dst[a]) *dst[a] = p[a];
    return BM25X_OK;
}

// A batch as one list of a device merge (bm25x_merged_search).
struct BatchList final : ListRun {
    bm25x_batch *b;
    explicit BatchList(bm25x_batch *b_) : b(b_) {}
    ~BatchList() override { bm25x_batch_destroy(b); }
    const ResultRows &rows() const override { return b->out; }
    cudaEvent_t done() const override { return b->ev1; }
    int add_stats(bm25x_search_stats *acc) override { return bm25x_batch_add_stats(b, acc); }
};

int bm25x_batch_list(bm25x_index *ix, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms, uint32_t k,
                     const uint8_t *allow, std::unique_ptr<ListRun> *out) {
    bm25x_batch *b = nullptr;
    const int rc = bm25x_batch_prepare(ix, nq, q_off, q_terms, k, allow, &b);
    if (rc != BM25X_OK) return rc;
    out->reset(new BatchList(b));
    return batch_enqueue(b, ix->stream, true);
}

// The figures of the batch's last timed run, added to *acc (bm25x_batch_run fills a zeroed one).
static int bm25x_batch_add_stats(bm25x_batch *b, bm25x_search_stats *acc) {
    BM25X_CUDA_TRY(cudaSetDevice(b->ix->device));
    float ms = 0.f;
    unsigned long long fetched = 0;
    BM25X_CUDA_TRY(cudaEventElapsedTime(&ms, b->ev0, b->ev1));
    BM25X_CUDA_TRY(cudaMemcpy(&fetched, b->d_fetched, sizeof(fetched), cudaMemcpyDeviceToHost));
    acc->kernel_ms += ms;
    acc->postings += b->postings;
    acc->bytes_algo += 8ull * b->postings + 8ull * (uint64_t)b->live * b->k + 16ull * b->qterms;
    acc->launches += b->launches;
    acc->queries += b->live;
    acc->postings_fetched += fetched;  // 0 for the CTA kernel (always exhaustive)
    return BM25X_OK;
}

// Large batches run as a pipeline of slices: while slice s is on the GPU the host canonicalises and uploads slice s + 1,
// and the results of slice s - 1 travel to the host on a second stream.  Same results, row for row.
static int search_batch_sliced(bm25x_index *ix, const SlicePlan &plan, const uint32_t *q_off, const uint32_t *q_terms,
                               uint32_t k, const uint8_t *allow, const ResultRows &host, bm25x_search_stats *stats) {
    using clk = std::chrono::steady_clock;
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    const uint32_t n_slices = plan.n;
    std::vector<bm25x_batch *> bs(n_slices, nullptr);
    std::vector<cudaEvent_t> done(n_slices, nullptr);
    int rc = BM25X_OK;
    double host_ms = 0.0;
    auto fail = [&](int code) {
        cudaStreamSynchronize(ix->stream);
        cudaStreamSynchronize(ix->copy_stream);
        for (uint32_t s = 0; s < n_slices; ++s) {
            if (done[s]) cudaEventDestroy(done[s]);
            if (bs[s]) bm25x_batch_destroy(bs[s]);
        }
        return code;
    };
    for (uint32_t s = 0; s < n_slices && rc == BM25X_OK; ++s) {
        const uint32_t a = plan.begin(s), e = plan.begin(s + 1);
        const auto t0 = clk::now();
        // (q_off + a holds absolute offsets into q_terms: the slice is prepared in place)
        rc = bm25x_batch_prepare(ix, e - a, q_off + a, q_terms, k, allow, &bs[s]);
        host_ms += std::chrono::duration<double, std::milli>(clk::now() - t0).count();
        if (rc != BM25X_OK) break;
        bm25x_batch *b = bs[s];
        rc = batch_enqueue(b, ix->stream, stats != nullptr);
        if (rc != BM25X_OK) break;
        cudaError_t ce = cudaEventCreateWithFlags(&done[s], cudaEventDisableTiming);
        if (ce == cudaSuccess) ce = cudaEventRecord(done[s], ix->stream);
        if (ce == cudaSuccess) ce = cudaStreamWaitEvent(ix->copy_stream, done[s], 0);
        if (ce == cudaSuccess) ce = b->out.copy_to(host.from(a, k), e - a, k, ix->copy_stream);
        if (ce != cudaSuccess) {
            bm25x_set_error("bm25x_search_batch (slice %u): %s", s, cudaGetErrorString(ce));
            return fail(BM25X_ERR_CUDA);
        }
    }
    if (rc != BM25X_OK) return fail(rc);
    const auto t2 = clk::now();
    cudaError_t ce = cudaStreamSynchronize(ix->copy_stream);  // every download (hence every kernel) has finished
    if (ce != cudaSuccess) {
        bm25x_set_error("bm25x_search_batch: %s", cudaGetErrorString(ce));
        return fail(BM25X_ERR_CUDA);
    }
    if (stats) {
        memset(stats, 0, sizeof(*stats));
        for (uint32_t s = 0; s < n_slices; ++s) {
            rc = bm25x_batch_add_stats(bs[s], stats);
            if (rc != BM25X_OK) return fail(rc);
        }
        stats->h2d_ms = host_ms;  // canonicalise + upload of all slices (overlapped with the kernels but for the first)
        stats->d2h_ms = std::chrono::duration<double, std::milli>(clk::now() - t2).count();  // wait for the last download
    }
    for (uint32_t s = 0; s < n_slices; ++s) {
        cudaEventDestroy(done[s]);
        bm25x_batch_destroy(bs[s]);
    }
    return BM25X_OK;
}

extern "C" int bm25x_search_batch(bm25x_index *ix, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                                  uint32_t k, const uint8_t *allow, uint32_t *out_doc, float *out_score,
                                  double *out_score64, uint16_t *out_payload, uint32_t *out_n,
                                  bm25x_search_stats *stats) {
    using clk = std::chrono::steady_clock;
    if (ix && q_off && k != 0) {
        const SlicePlan plan(ix->slice_min, nq);
        if (plan.n > 1)
            return search_batch_sliced(ix, plan, q_off, q_terms, k, allow,
                                       {out_doc, out_score, out_score64, out_payload, out_n}, stats);
    }
    bm25x_batch *b = nullptr;
    const auto t0 = clk::now();
    int rc = bm25x_batch_prepare(ix, nq, q_off, q_terms, k, allow, &b);
    if (rc != BM25X_OK) return rc;
    if (stats) cudaStreamSynchronize(ix->stream);  // so that h2d_ms means what it says (costs nothing: run follows)
    const auto t1 = clk::now();
    rc = bm25x_batch_run(b, nullptr, stats);  // stats == NULL: asynchronous, the fetch below synchronises
    const auto t2 = clk::now();
    if (rc == BM25X_OK) rc = bm25x_batch_fetch(b, out_doc, out_score, out_score64, out_payload, out_n);
    if (stats && rc == BM25X_OK) {  // host-clock phases of this call: canonicalise + upload, download
        stats->h2d_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
        stats->d2h_ms = std::chrono::duration<double, std::milli>(clk::now() - t2).count();
    }
    bm25x_batch_destroy(b);
    return rc;
}

// ---- sealed + growing segment (search.rs:83-135 then :137-282 share one Results heap): both top-k lists, merged ----
extern "C" int bm25x_merge_topk(uint32_t nq, uint32_t k, const uint32_t *doc_a, const float *score_a,
                                const double *score64_a, const uint16_t *payload_a, const uint32_t *n_a,
                                const uint32_t *doc_b, const float *score_b, const double *score64_b,
                                const uint16_t *payload_b, const uint32_t *n_b, uint32_t doc_base_b, uint32_t *out_doc,
                                float *out_score, double *out_score64, uint16_t *out_payload, uint32_t *out_n) {
    if (const int rc = check_k(k, false); rc != BM25X_OK) return rc;
    if (nq && (!doc_a || !score64_a || !n_a || !doc_b || !score64_b || !n_b || !out_doc || !out_n) ||
        (out_score && (!score_a || !score_b)) || (out_payload && (!payload_a || !payload_b))) {
        bm25x_set_error("bm25x_merge_topk: null argument (f64 scores of both lists are required)");
        return BM25X_ERR_INVALID;
    }
    // a shifted b id must stay a real doc id: BM25X_DOC_INF marks empty slots, and a wrapped sum would name another document
    for (uint32_t q = 0; q < nq; q++)
        for (uint32_t i = 0, nb = std::min(n_b[q], k); i < nb; i++)
            if ((uint64_t)doc_b[(size_t)q * k + i] + doc_base_b > (uint64_t)BM25X_DOC_INF - 2u) {
                bm25x_set_error("bm25x_merge_topk: doc %u of list b + doc_base_b %u exceeds the largest doc id %u",
                                doc_b[(size_t)q * k + i], doc_base_b, BM25X_DOC_INF - 2u);
                return BM25X_ERR_INVALID;
            }
#pragma omp parallel for schedule(static) num_threads(nq < 4096 ? 1 : bm25x_host_threads(16))
    for (uint32_t q = 0; q < nq; q++) {
        const size_t base = (size_t)q * k;
        const uint32_t na = std::min(n_a[q], k), nb = std::min(n_b[q], k);
        uint32_t ia = 0, ib = 0, o = 0;
        while (o < k && (ia < na || ib < nb)) {
            // score desc; on equal scores list a first: its doc ids are all below doc_base_b (canonical doc-id order)
            const bool take_a = ib >= nb || (ia < na && score64_a[base + ia] >= score64_b[base + ib]);
            const size_t src = base + (take_a ? ia : ib);
            out_doc[base + o] = take_a ? doc_a[src] : doc_b[src] + doc_base_b;
            if (out_score) out_score[base + o] = take_a ? score_a[src] : score_b[src];
            if (out_score64) out_score64[base + o] = take_a ? score64_a[src] : score64_b[src];
            if (out_payload)
                for (int c = 0; c < 3; c++)
                    out_payload[(base + o) * 3 + c] = take_a ? payload_a[src * 3 + c] : payload_b[src * 3 + c];
            take_a ? ia++ : ib++;
            o++;
        }
        out_n[q] = o;
        for (; o < k; o++) {
            out_doc[base + o] = BM25X_DOC_INF;
            if (out_score) out_score[base + o] = 0.f;
            if (out_score64) out_score64[base + o] = 0.0;
            if (out_payload) out_payload[(base + o) * 3] = out_payload[(base + o) * 3 + 1] = out_payload[(base + o) * 3 + 2] = 0;
        }
    }
    return BM25X_OK;
}

extern "C" int bm25x_search_batch_growing(bm25x_index *sealed, bm25x_index *growing, uint32_t nq, const uint32_t *q_off,
                                          const uint32_t *q_terms, uint32_t k, const uint8_t *allow_sealed,
                                          const uint8_t *allow_growing, uint32_t *out_doc, float *out_score,
                                          double *out_score64, uint16_t *out_payload, uint32_t *out_n,
                                          bm25x_search_stats *stats) {
    if (growing) {
        if (!sealed || sealed->d.n_terms != growing->d.n_terms || sealed->device != growing->device) {
            bm25x_set_error("bm25x_search_batch_growing: the growing segment does not belong to this sealed index");
            return BM25X_ERR_INVALID;
        }
        if (const int rc = check_k(k, false); rc != BM25X_OK) return rc;
    }
    // both top-k lists merged on the device: equal scores keep the sealed list first (its ids are all below the base).
    // stats->queries is the sealed search's: a growing live query is a sealed one.
    SealedSide side;
    side.ix = sealed;
    SideFilter f;
    f.allow_sealed = allow_sealed;
    f.allow_growing = allow_growing;
    return sealed_side_search("bm25x_search_batch_growing", side, growing, f, false, nq, q_off, q_terms, k,
                              {out_doc, out_score, out_score64, out_payload, out_n}, stats,
                              std::chrono::steady_clock::now());
}
