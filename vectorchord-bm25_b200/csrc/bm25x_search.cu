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

#include "bm25x_common.h"

#include "bm25x_device.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// bm25::evaluate (crates/bm25/src/evaluate.rs:22-74): one thread per (document, query) pair.
__global__ void k_evaluate(uint32_t n_pairs, const uint32_t *__restrict__ d_off, const uint32_t *__restrict__ d_terms,
                           const uint32_t *__restrict__ d_tfs, const uint32_t *__restrict__ q_off,
                           const uint32_t *__restrict__ q_terms, const uint32_t *__restrict__ fn_len,
                           const double *__restrict__ idf, const double *__restrict__ s1d, const uint32_t *__restrict__ df,
                           uint32_t n_terms, double k1, double *__restrict__ out) {
    uint32_t pidx = blockIdx.x * blockDim.x + threadIdx.x;
    if (pidx >= n_pairs) return;
    uint32_t a = d_off[pidx], b = d_off[pidx + 1];
    uint64_t len = 0;  // Document::length(): saturating Σ tf (vector.rs:77-83)
    for (uint32_t i = a; i < b; ++i) {
        len += d_tfs[i];
        if (len > 0xFFFFFFFFull) len = 0xFFFFFFFFull;
    }
    int lo = 0, hi = 256;  // length_to_fieldnorm, bm25.rs:278-283
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (fn_len[mid] <= (uint32_t)len) lo = mid + 1;
        else hi = mid;
    }
    const int fn = lo - 1;
    uint32_t cursor = a;
    double result = 0.0;
    const double k1p1 = __dadd_rn(k1, 1.0);
    for (uint32_t qi = q_off[pidx]; qi < q_off[pidx + 1]; ++qi) {
        uint32_t key = q_terms[qi];
        while (cursor < b && d_terms[cursor] < key) cursor++;
        if (!(cursor < b && d_terms[cursor] == key)) continue;
        if (key >= n_terms || df[key] == 0) continue;  // address_tokens::read → None
        double tfd = (double)d_tfs[cursor];
        double tfv = __ddiv_rn(__dmul_rn(tfd, k1p1), __dadd_rn(tfd, s1d[fn]));  // bm25.rs:291-295
        result = __dadd_rn(result, __dmul_rn(idf[key], tfv));
    }
    out[pidx] = result;
}

}  // namespace

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

// Canonicalises the queries (bm25x_canonicalise), groups them by term-count class and uploads everything with ONE copy
// from a page-locked staging buffer cached in the index handle.
extern "C" int bm25x_batch_prepare(bm25x_index *ix, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                                   uint32_t k, const uint8_t *allow, bm25x_batch **out) {
    if (!ix || !out || (nq && (!q_off || (!q_terms && q_off[nq] != 0)))) {
        bm25x_set_error("bm25x_batch_prepare: null argument");
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    if (ix->h_df.size() != ix->d.n_terms) {
        bm25x_set_error("bm25x_batch_prepare: replica not finalized (bm25x_index_finalize_replica)");
        return BM25X_ERR_INVALID;
    }
    if (k == 0) {
        bm25x_set_error("number of needed rows is set to 0");  // scanners/default.rs:114-116
        return BM25X_ERR_LIMIT_ZERO;
    }
    if (k > BM25X_MAX_K) {
        bm25x_set_error("bm25x_batch_prepare: k=%u > BM25X_MAX_K=%d", k, BM25X_MAX_K);
        return BM25X_ERR_UNSUPPORTED;
    }
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
    if (ix->h_stage_words < words) {
        if (ix->h_stage) {
            cudaStreamSynchronize(st);  // an earlier batch's upload may still read it
            cudaFreeHost(ix->h_stage);
        }
        ix->h_stage = nullptr;
        ix->h_stage_words = 0;
        const size_t cap = words + words / 4 + 1024;
        e = cudaMallocHost((void **)&ix->h_stage, cap * sizeof(uint32_t));
        if (e != cudaSuccess) {
            bm25x_set_error("bm25x_batch_prepare: page-locked staging buffer: %s", cudaGetErrorString(e));
            delete b;
            return BM25X_ERR_OOM;
        }
        ix->h_stage_words = cap;
    } else if (ix->h_stage_busy) {
        cudaEventSynchronize(ix->h_stage_free);  // the previous upload from this buffer has been issued; wait for it
    }
    uint32_t *hs = ix->h_stage;
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
    e = cudaMemcpyAsync(d_q, hs, words * sizeof(uint32_t), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        if (!ix->h_stage_free) e = cudaEventCreateWithFlags(&ix->h_stage_free, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventRecord(ix->h_stage_free, st);
        ix->h_stage_busy = true;
    }
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

// The launches of one run on st, counted in b->launches.  Timed: the fetched-postings counter is zeroed and the run sits
// between the batch's events ev0 and ev1.  Does not synchronise.
static int batch_enqueue(bm25x_batch *b, cudaStream_t st, bool timed) {
    bm25x_index *ix = b->ix;
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    b->last_stream = (void *)st;
    if (st != ix->stream) BM25X_CUDA_TRY(cudaStreamWaitEvent(st, b->ev_ready, 0));  // uploads were issued on the library's stream
    const DeviceIndex &d = ix->d;
    uint32_t launches = 0;
    if (timed) {
        BM25X_CUDA_TRY(cudaMemsetAsync(b->d_fetched, 0, sizeof(unsigned long long), st));
        BM25X_CUDA_TRY(cudaEventRecord(b->ev0, st));
    }
    for (int c = 0; c < kNumClasses; ++c) {
        Group &g = b->groups[c];
        if (!g.nq) continue;
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
        sp.fetched = b->d_fetched;
        sp.n_docs = d.n_docs;
        sp.q_ids = g.d_ids;
        sp.q_off = g.d_off;
        sp.q_terms = g.d_terms;
        sp.nq = g.nq;
        sp.k = b->k;
        sp.allow = b->d_allow;
        sp.work_counter = g.d_counter;
        sp.out_doc = b->out.doc;
        sp.out_score = b->out.score;
        sp.out_score64 = b->out.score64;
        sp.out_payload = b->out.payload;
        sp.out_n = b->out.n;
        BM25X_CUDA_TRY(cudaMemsetAsync(g.d_counter, 0, sizeof(int), st));
        sp.q2 = g.d_q2;
        sp.resume = g.d_resume;
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

const ResultRows &bm25x_batch_rows(const bm25x_batch *b) { return b->out; }

// An asynchronous timed run on the index's stream (the slices of search_batch_sliced, the shards of
// bm25x_sharded_search_batch); bm25x_batch_add_stats reads its figures once it has finished.
int bm25x_batch_run_timed(bm25x_batch *b) { return batch_enqueue(b, b->ix->stream, true); }

cudaEvent_t bm25x_batch_done_event(bm25x_batch *b) { return b->ev1; }

// The figures of the batch's last timed run, added to *acc (bm25x_batch_run fills a zeroed one).
int bm25x_batch_add_stats(bm25x_batch *b, bm25x_search_stats *acc) {
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
    if (k == 0) {
        bm25x_set_error("number of needed rows is set to 0");
        return BM25X_ERR_LIMIT_ZERO;
    }
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

// Two searches of the same queries (sealed, growing) as one: times and work add up, `queries` is the first one's.
static void add_work(bm25x_search_stats *out, const bm25x_search_stats &a, const bm25x_search_stats &b) {
    *out = a;
    out->kernel_ms += b.kernel_ms;
    out->h2d_ms += b.h2d_ms;
    out->d2h_ms += b.d2h_ms;
    out->postings += b.postings;
    out->bytes_algo += b.bytes_algo;
    out->launches += b.launches;
    out->postings_fetched += b.postings_fetched;
}

extern "C" int bm25x_search_batch_growing(bm25x_index *sealed, bm25x_index *growing, uint32_t nq, const uint32_t *q_off,
                                          const uint32_t *q_terms, uint32_t k, const uint8_t *allow_sealed,
                                          const uint8_t *allow_growing, uint32_t *out_doc, float *out_score,
                                          double *out_score64, uint16_t *out_payload, uint32_t *out_n,
                                          bm25x_search_stats *stats) {
    if (!growing)
        return bm25x_search_batch(sealed, nq, q_off, q_terms, k, allow_sealed, out_doc, out_score, out_score64,
                                  out_payload, out_n, stats);
    if (!sealed || sealed->d.n_terms != growing->d.n_terms || sealed->device != growing->device) {
        bm25x_set_error("bm25x_search_batch_growing: the growing segment does not belong to this sealed index");
        return BM25X_ERR_INVALID;
    }
    if (k == 0) {
        bm25x_set_error("number of needed rows is set to 0");
        return BM25X_ERR_LIMIT_ZERO;
    }
    const size_t slots = (size_t)nq * k;
    std::vector<uint32_t> doc[2], n[2];
    std::vector<float> sc[2];
    std::vector<double> sc64[2];
    std::vector<uint16_t> pay[2];
    bm25x_search_stats st[2];
    bm25x_index *seg[2] = {sealed, growing};
    const uint8_t *allow[2] = {allow_sealed, allow_growing};
    for (int s = 0; s < 2; s++) {
        doc[s].resize(slots ? slots : 1);
        n[s].resize(nq ? nq : 1);
        sc[s].resize(slots ? slots : 1);
        sc64[s].resize(slots ? slots : 1);
        if (out_payload) pay[s].resize(slots ? slots * 3 : 1);
        const int rc = bm25x_search_batch(seg[s], nq, q_off, q_terms, k, allow[s], doc[s].data(), sc[s].data(),
                                          sc64[s].data(), out_payload ? pay[s].data() : nullptr, n[s].data(), &st[s]);
        if (rc != BM25X_OK) return rc;
    }
    if (stats) add_work(stats, st[0], st[1]);
    return bm25x_merge_topk(nq, k, doc[0].data(), sc[0].data(), sc64[0].data(), out_payload ? pay[0].data() : nullptr,
                            n[0].data(), doc[1].data(), sc[1].data(), sc64[1].data(),
                            out_payload ? pay[1].data() : nullptr, n[1].data(), sealed->d.n_docs, out_doc, out_score,
                            out_score64, out_payload, out_n);
}

// ---------------------------------------------------------------------------------------------
uint32_t bm25x_fieldnorm_to_length(uint8_t fn);

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
    if (!ix || (n_pairs && (!d_off || !q_off || !out))) {
        bm25x_set_error("bm25x_evaluate_batch: null argument");
        return BM25X_ERR_INVALID;
    }
    if (n_pairs == 0) return BM25X_OK;
    if (d_off[n_pairs] != 0 && !d_tfs) {
        bm25x_set_error("bm25x_evaluate_batch: null argument");
        return BM25X_ERR_INVALID;
    }
    {   // Document / Query invariants (vector.rs:46-134)
        int vrc = bm25x_check_vectors(n_pairs, d_off, d_terms, d_tfs);
        if (vrc == BM25X_OK) vrc = bm25x_check_vectors(n_pairs, q_off, q_terms, nullptr);
        if (vrc != BM25X_OK) return vrc;
    }
    if (ix->h_df.size() != ix->d.n_terms) {
        bm25x_set_error("bm25x_evaluate_batch: replica not finalized (bm25x_index_finalize_replica)");
        return BM25X_ERR_INVALID;
    }
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    const uint32_t nd = d_off[n_pairs], nqt = q_off[n_pairs];
    const uint32_t T = ix->d.n_terms;
    {   // idf table (bm25.rs:285-289) with the host libm, like the reference's f64::ln, and the fieldnorm -> length table:
        // they depend on the index alone — built once, kept on the device (freed with the handle)
        std::lock_guard<std::mutex> lk(ix->eval_mutex);
        if (!ix->eval_idf) {
            std::vector<double> h_idf(T ? T : 1);
            for (uint32_t t = 0; t < T; ++t)
                h_idf[t] = log(((double)ix->d.n_docs + 1.0) / ((double)ix->h_df[t] + 0.5));
            uint32_t h_fn[256];
            for (int f = 0; f < 256; ++f) h_fn[f] = bm25x_fieldnorm_to_length((uint8_t)f);
            double *d_idf = nullptr;
            uint32_t *d_fn = nullptr;
            BM25X_CUDA_TRY(cudaMalloc((void **)&d_idf, 8 * (size_t)(T ? T : 1)));
            ix->allocs.push_back((void *)d_idf);
            BM25X_CUDA_TRY(cudaMalloc((void **)&d_fn, sizeof(h_fn)));
            ix->allocs.push_back((void *)d_fn);
            BM25X_CUDA_TRY(cudaMemcpy(d_idf, h_idf.data(), 8 * (size_t)(T ? T : 1), cudaMemcpyHostToDevice));
            BM25X_CUDA_TRY(cudaMemcpy(d_fn, h_fn, sizeof(h_fn), cudaMemcpyHostToDevice));
            ix->eval_fn_len = d_fn;
            ix->eval_idf = d_idf;
        }
    }
    uint32_t *g_doff = nullptr, *g_dt = nullptr, *g_df = nullptr, *g_qoff = nullptr, *g_qt = nullptr;
    uint32_t *const g_fn = ix->eval_fn_len;
    double *const g_idf = ix->eval_idf;
    double *g_out = nullptr;
    int rc = BM25X_OK;
    cudaError_t e = cudaSuccess;
    auto A = [&](void **p, size_t bytes) {
        if (e == cudaSuccess) e = cudaMalloc(p, bytes ? bytes : 4);
    };
    A((void **)&g_doff, 4 * ((size_t)n_pairs + 1));
    A((void **)&g_dt, 4 * (size_t)nd);
    A((void **)&g_df, 4 * (size_t)nd);
    A((void **)&g_qoff, 4 * ((size_t)n_pairs + 1));
    A((void **)&g_qt, 4 * (size_t)nqt);
    A((void **)&g_out, 8 * (size_t)n_pairs);
    auto H = [&](void *dst, const void *src, size_t bytes) {
        if (e == cudaSuccess && bytes) e = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
    };
    H(g_doff, d_off, 4 * ((size_t)n_pairs + 1));
    H(g_dt, d_terms, 4 * (size_t)nd);
    H(g_df, d_tfs, 4 * (size_t)nd);
    H(g_qoff, q_off, 4 * ((size_t)n_pairs + 1));
    H(g_qt, q_terms, 4 * (size_t)nqt);
    if (e == cudaSuccess) {
        k_evaluate<<<(n_pairs + 127) / 128, 128>>>(n_pairs, g_doff, g_dt, g_df, g_qoff, g_qt, g_fn, g_idf, ix->d.s1d,
                                                   ix->d.df, T, ix->k1, g_out);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(out, g_out, 8 * (size_t)n_pairs, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) {
        bm25x_set_error("bm25x_evaluate_batch: %s", cudaGetErrorString(e));
        rc = BM25X_ERR_CUDA;
    }
    cudaFree(g_doff);
    cudaFree(g_dt);
    cudaFree(g_df);
    cudaFree(g_qoff);
    cudaFree(g_qt);
    cudaFree(g_out);
    return rc;
}
