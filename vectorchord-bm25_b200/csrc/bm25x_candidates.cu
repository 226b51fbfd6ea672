// bm25x_candidates.cu — per-query candidate lists (bm25x_search_candidates, DESIGN §4.8): each query's top-k over its own
// doc ids, scored by posting lookups instead of streamed lists.
//
// The reference's bm25::search (crates/bm25/src/search.rs:28-36) takes the filter of one index scan, and every scan
// carries its own WHERE clause and bm25.prefilter (src/index/fetcher.rs:181-215); the batch ABI's single `allow` bitmap
// flattens that.  Here every query of a batch brings its own candidate list, the form a filter or an ANN pre-selection
// (hybrid retrieval) hands over: a short list is cheaper to answer by looking each candidate up in each term's list than
// by streaming every list.
//
// One call on the index's stream:
//   1. one upload: the canonical queries (live terms ascending) and the candidate lists of the live queries;
//   2. CUB segmented sort of every query's candidates by doc id: neighbouring threads read neighbouring block-table
//      entries and blocks, and duplicates become adjacent;
//   3. k_cand_lookup: one thread per candidate.  Per live term in ascending order the block table (SummaryTuple min doc),
//      then the 128-posting block (probe_block / probe_in_block, shared with the search kernel's probes), the f64 sum in
//      the reference's operation order.  Key = f64 score bits + 1 (0: no live term, or a duplicate);
//   4. CUB stable segmented sort of the keys descending, the doc ids riding along: equal scores keep doc ids ascending;
//   5. k_cand_rows: the first min(k, matches) entries of every query into its result row.
// Rows are bit for bit those of bm25x_search_batch with the bitmap of the query's candidates: both are the exact
// (f64 score desc, doc asc) order of the matching documents.
#include <limits.h>
#include <string.h>

#include <chrono>
#include <cub/device/device_segmented_sort.cuh>
#include <vector>

#include "bm25x_common.h"
#include "bm25x_device.cuh"

namespace {

// The query of candidate slot i: the last q < nq with off[q] <= i (off[0] = 0 <= i < off[nq]; empty queries are skipped).
__device__ __forceinline__ uint32_t query_of(const uint32_t *__restrict__ off, uint32_t nq, uint32_t i) {
    uint32_t lo = 0, hi = nq - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (__ldg(&off[mid]) <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// One thread per sorted candidate: its key (f64 score bits + 1; 0 when it holds no live term or repeats the previous
// candidate).  p.fetched += block-table entries and postings read.
__global__ void __launch_bounds__(256) k_cand_lookup(const SearchParams p, const uint32_t *__restrict__ q_off,
                                                     const uint32_t *__restrict__ q_terms, const uint32_t *__restrict__ c_off,
                                                     uint32_t nq, const uint32_t *__restrict__ docs, uint32_t n,
                                                     uint64_t *__restrict__ key) {
    uint32_t steps = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t q = query_of(c_off, nq, i);
        const uint32_t doc = docs[i];
        uint64_t kv = 0;
        if (i == __ldg(&c_off[q]) || docs[i - 1] != doc) {
            double sx = 0.0;
            bool hit = false;
            for (uint32_t j = __ldg(&q_off[q]), e = __ldg(&q_off[q + 1]); j < e; ++j) {  // ascending term ids
                const uint32_t t = __ldg(&q_terms[j]);
                const uint32_t dft = __ldg(&p.df[t]);
                const uint32_t l = probe_block(p, __ldg(&p.blk_off[t]), (dft + BM25X_BLOCK - 1) / BM25X_BLOCK, doc, steps);
                const uint32_t w = l > 0u ? probe_in_block(p, __ldg(&p.post_off[t]), dft, l - 1u, doc, steps) : 0u;
                if (w) {
                    sx = __dadd_rn(sx, score_f64(w, __ldg(&p.s0d[t]), p.s1d));
                    hit = true;
                }
            }
            if (hit) kv = (uint64_t)__double_as_longlong(sx) + 1u;  // scores are >= 0: the bits are monotone
        }
        key[i] = kv;
    }
    unsigned long long f = steps;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) f += __shfl_xor_sync(0xFFFFFFFFu, f, o);
    if ((threadIdx.x & 31) == 0 && f) atomicAdd(p.fetched, f);
}

// One thread per entry of the keys sorted descending: entry r < k of query q with a non-zero key is slot r of row q.  The
// thread of entry 0 writes n[q] = min(k, matching entries).  Slots past n keep the reset of the rows.
__global__ void __launch_bounds__(256) k_cand_rows(const uint16_t *__restrict__ payload, const uint32_t *__restrict__ c_off,
                                                   uint32_t nq, const uint64_t *__restrict__ key,
                                                   const uint32_t *__restrict__ doc, uint32_t n, uint32_t k, ResultRows out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t q = query_of(c_off, nq, i);
        const uint32_t a = __ldg(&c_off[q]), r = i - a;
        if (r >= k) continue;
        const uint64_t kv = key[i];
        const size_t o = (size_t)q * k + r;
        if (kv) {
            const uint32_t d = doc[i];
            const double sc = __longlong_as_double((long long)(kv - 1u));
            out.doc[o] = d;
            out.score[o] = (float)sc;
            out.score64[o] = sc;
            out.payload[o * 3 + 0] = payload[(size_t)d * 3 + 0];
            out.payload[o * 3 + 1] = payload[(size_t)d * 3 + 1];
            out.payload[o * 3 + 2] = payload[(size_t)d * 3 + 2];
        }
        if (r == 0) {
            uint32_t lo = a, hi = __ldg(&c_off[q + 1]);  // first entry without a match
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (key[mid] != 0u) lo = mid + 1;
                else hi = mid;
            }
            out.n[q] = min(lo - a, k);
        }
    }
}

// A prepared candidate search of one handle: its device inputs, scratch and rows, freed with it.
struct CandBatch final : ListRun {
    bm25x_index *ix = nullptr;
    uint32_t nq = 0, k = 0;
    uint32_t n_cand = 0;          // candidates of the live queries
    uint32_t live = 0, launches = 0;
    uint64_t postings = 0, qterms = 0, lookups = 0;
    uint32_t *d_q_off = nullptr, *d_q_terms = nullptr, *d_c_off = nullptr, *d_docs[2] = {nullptr, nullptr};
    uint64_t *d_key[2] = {nullptr, nullptr};
    void *d_temp = nullptr;
    size_t temp_bytes = 0;
    unsigned long long *d_fetched = nullptr;
    ResultRows out;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<void *> allocs;

    ~CandBatch() override {
        cudaSetDevice(ix->device);
        for (void *p : allocs) cudaFreeAsync(p, ix->stream);
        out.release(ix->stream);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    }
    const ResultRows &rows() const override { return out; }
    cudaEvent_t done() const override { return ev1; }
    int add_stats(bm25x_search_stats *acc) override {
        BM25X_CUDA_TRY(cudaSetDevice(ix->device));
        float ms = 0.f;
        unsigned long long fetched = 0;
        BM25X_CUDA_TRY(cudaEventElapsedTime(&ms, ev0, ev1));
        BM25X_CUDA_TRY(cudaMemcpy(&fetched, d_fetched, sizeof(fetched), cudaMemcpyDeviceToHost));
        acc->kernel_ms += ms;
        acc->postings += postings;
        acc->bytes_algo += 8ull * lookups + 8ull * (uint64_t)live * k + 16ull * qterms;
        acc->launches += launches;
        acc->queries += live;
        acc->postings_fetched += fetched;
        return BM25X_OK;
    }
    template <typename T>
    cudaError_t alloc(T **p, size_t n) {
        const cudaError_t e = cudaMallocAsync((void **)p, sizeof(T) * (n ? n : 1), ix->stream);
        if (e == cudaSuccess) allocs.push_back((void *)*p);
        return e;
    }
};

// The request checks, canonicalisation and one upload of bm25x_search_candidates; rows reset, nothing run.
int cand_prepare(const char *who, bm25x_index *ix, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                 const uint32_t *c_off, const uint32_t *c_docs, uint32_t k, std::unique_ptr<CandBatch> *out) {
    if (!ix) {
        bm25x_set_error("bm25x_batch_prepare: null argument");
        return BM25X_ERR_INVALID;
    }
    if (const int rc = check_queries(nq, q_off, q_terms); rc != BM25X_OK) return rc;
    if (nq && (!c_off || (!c_docs && c_off[nq] != 0))) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    if (ix->h_df.size() != ix->d.n_terms) {
        bm25x_set_error("bm25x_batch_prepare: replica not finalized (bm25x_index_finalize_replica)");
        return BM25X_ERR_INVALID;
    }
    if (const int rc = check_k(k, true); rc != BM25X_OK) return rc;
    const uint32_t *h_df = ix->h_df.data();
    CanonQueries cq;
    if (const int rc = bm25x_canonicalise(h_df, ix->d.n_terms, nq, q_off, q_terms, &cq); rc != BM25X_OK) return rc;
    if (const int rc = check_candidates(who, nq, c_off, c_docs, ix->d.n_docs); rc != BM25X_OK) return rc;
    const size_t qbase = nq ? q_off[0] : 0;
    uint32_t *const canon = cq.terms.get(), *const live = cq.live.get();
    // ---- the upload's layout: [q_off' nq+1 | q_terms' | c_off' nq+1 | candidates]; a query without a live term has
    // no candidate ----
    std::unique_ptr<CandBatch> b(new CandBatch());
    b->ix = ix;
    b->nq = nq;
    b->k = k;
    std::vector<uint32_t> qo(nq + 1, 0), co(nq + 1, 0);
    uint64_t n_cand = 0;
    for (uint32_t i = 0; i < nq; i++) {
        const uint32_t m = live[i], nc = m ? c_off[i + 1] - c_off[i] : 0u;
        qo[i + 1] = qo[i] + m;
        n_cand += nc;
        if (n_cand > (uint64_t)INT_MAX) {
            bm25x_set_error("%s: more than %d candidates in one call", who, INT_MAX);
            return BM25X_ERR_UNSUPPORTED;
        }
        co[i + 1] = (uint32_t)n_cand;
        if (m) {
            b->live++;
            b->qterms += m;
            uint64_t df_sum = 0;
            for (uint32_t j = 0; j < m; j++) df_sum += h_df[canon[q_off[i] - qbase + j]];
            b->postings += df_sum;
            b->lookups += (uint64_t)nc * m;
        }
    }
    if (nq > (uint32_t)INT_MAX) {
        bm25x_set_error("%s: more than %d queries in one call", who, INT_MAX);
        return BM25X_ERR_UNSUPPORTED;
    }
    b->n_cand = (uint32_t)n_cand;
    const size_t words = 2 * ((size_t)nq + 1) + qo[nq] + n_cand;
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    std::lock_guard<std::mutex> stage_lock(ix->stage_mutex);  // the staging buffer is shared by the uploads of this index
    uint32_t *hs = nullptr;
    if (const int rc = stage_reserve(ix, who, words, &hs); rc != BM25X_OK) return rc;
    uint32_t *hq_terms = hs + nq + 1, *hc_off = hq_terms + qo[nq], *hdocs = hc_off + nq + 1;
    std::copy(qo.begin(), qo.end(), hs);
    std::copy(co.begin(), co.end(), hc_off);
    const int nthr = nq < 4096 ? 1 : bm25x_host_threads(16);
#pragma omp parallel for schedule(dynamic, 256) num_threads(nthr)
    for (uint32_t i = 0; i < nq; i++) {
        const uint32_t m = live[i];
        if (!m) continue;
        uint32_t *t = hq_terms + qo[i];
        std::copy(canon + (q_off[i] - qbase), canon + (q_off[i] - qbase) + m, t);
        if (m > 32) std::sort(t, t + m);  // canonical order is rarest-32-first; the sum runs over ascending term ids
        std::copy(c_docs + c_off[i], c_docs + c_off[i + 1], hdocs + co[i]);
    }
    cudaError_t e = b->alloc(&b->d_q_off, words);
    if (e == cudaSuccess) e = stage_upload(ix, b->d_q_off, words);
    b->d_q_terms = b->d_q_off + nq + 1;
    b->d_c_off = b->d_q_terms + qo[nq];
    b->d_docs[0] = b->d_c_off + nq + 1;
    if (n_cand) {
        size_t t_docs = 0, t_keys = 0;
        cub::DoubleBuffer<uint32_t> dd(nullptr, nullptr);
        cub::DoubleBuffer<uint64_t> kk(nullptr, nullptr);
        if (e == cudaSuccess)
            e = cub::DeviceSegmentedSort::SortKeys(nullptr, t_docs, dd, (int)n_cand, (int)nq, b->d_c_off,
                                                   b->d_c_off + 1, ix->stream);
        if (e == cudaSuccess)
            e = cub::DeviceSegmentedSort::StableSortPairsDescending(nullptr, t_keys, kk, dd, (int)n_cand, (int)nq,
                                                                    b->d_c_off, b->d_c_off + 1, ix->stream);
        b->temp_bytes = std::max(t_docs, t_keys);
        if (e == cudaSuccess) e = b->alloc((uint8_t **)&b->d_temp, b->temp_bytes);
        if (e == cudaSuccess) e = b->alloc(&b->d_docs[1], n_cand);
        if (e == cudaSuccess) e = b->alloc(&b->d_key[0], n_cand);
        if (e == cudaSuccess) e = b->alloc(&b->d_key[1], n_cand);
    }
    if (e == cudaSuccess) e = b->alloc(&b->d_fetched, 1);
    if (e == cudaSuccess) e = b->out.alloc(nq, k, ix->stream);
    if (e == cudaSuccess) e = b->out.reset(nq, k, ix->stream);
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&b->ev1);
    if (e != cudaSuccess) {
        bm25x_set_error("%s: %s", who, cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? BM25X_ERR_OOM : BM25X_ERR_CUDA;
    }
    *out = std::move(b);
    return BM25X_OK;
}

// The run on ix's stream between the batch's events, without synchronising.
int cand_enqueue(CandBatch *b) {
    bm25x_index *ix = b->ix;
    const cudaStream_t st = ix->stream;
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    BM25X_CUDA_TRY(cudaMemsetAsync(b->d_fetched, 0, sizeof(unsigned long long), st));
    BM25X_CUDA_TRY(cudaEventRecord(b->ev0, st));
    b->launches = 0;
    if (b->n_cand) {
        const int n = (int)b->n_cand, nq = (int)b->nq;
        cub::DoubleBuffer<uint32_t> dd(b->d_docs[0], b->d_docs[1]);
        BM25X_CUDA_TRY(cub::DeviceSegmentedSort::SortKeys(b->d_temp, b->temp_bytes, dd, n, nq, b->d_c_off,
                                                          b->d_c_off + 1, st));
        const uint32_t grid = (uint32_t)std::min<uint64_t>(((uint64_t)n + 255) / 256, (uint64_t)ix->sm_count * 8);
        SearchParams sp = index_params(ix);
        sp.fetched = b->d_fetched;
        k_cand_lookup<<<grid, 256, 0, st>>>(sp, b->d_q_off, b->d_q_terms, b->d_c_off, b->nq, dd.Current(), b->n_cand,
                                            b->d_key[0]);
        BM25X_CUDA_TRY(cudaGetLastError());
        cub::DoubleBuffer<uint64_t> kk(b->d_key[0], b->d_key[1]);
        BM25X_CUDA_TRY(cub::DeviceSegmentedSort::StableSortPairsDescending(b->d_temp, b->temp_bytes, kk, dd, n, nq,
                                                                           b->d_c_off, b->d_c_off + 1, st));
        k_cand_rows<<<grid, 256, 0, st>>>(ix->d.payload, b->d_c_off, b->nq, kk.Current(), dd.Current(), b->n_cand, b->k,
                                          b->out);
        BM25X_CUDA_TRY(cudaGetLastError());
        b->launches = 4;  // two segmented sorts (counted once each), the lookups, the rows
    }
    BM25X_CUDA_TRY(cudaEventRecord(b->ev1, st));
    return BM25X_OK;
}

}  // namespace

int check_candidates(const char *who, uint32_t nq, const uint32_t *c_off, const uint32_t *c_docs, uint64_t n_ids) {
    // every offset before any entry: an offset that goes backwards must not lead the id check past the list's end
    for (uint32_t i = 0; i < nq; i++)
        if (c_off[i + 1] < c_off[i]) {
            bm25x_set_error("%s: c_off not monotone at %u", who, i);
            return BM25X_ERR_INVALID;
        }
    if (nq && c_off[nq] != c_off[0] && !c_docs) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    for (uint32_t i = 0; i < nq; i++)
        for (uint32_t j = c_off[i]; j < c_off[i + 1]; j++)
            if (c_docs[j] >= n_ids) {
                bm25x_set_error("%s: query %u, candidate entry %u: doc id %u >= n_docs %llu", who, i, j, c_docs[j],
                                (unsigned long long)n_ids);
                return BM25X_ERR_INVALID;
            }
    return BM25X_OK;
}

int cand_list(const char *who, bm25x_index *ix, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
              const uint32_t *c_off, const uint32_t *c_docs, uint32_t k, std::unique_ptr<ListRun> *out) {
    std::unique_ptr<CandBatch> b;
    const int rc = cand_prepare(who, ix, nq, q_off, q_terms, c_off, c_docs, k, &b);
    if (rc != BM25X_OK) return rc;
    CandBatch *raw = b.get();
    *out = std::move(b);
    return cand_enqueue(raw);
}

extern "C" int bm25x_search_candidates(bm25x_index *ix, uint32_t nq, const uint32_t *q_off, const uint32_t *q_terms,
                                       const uint32_t *c_off, const uint32_t *c_docs, uint32_t k, uint32_t *out_doc,
                                       float *out_score, double *out_score64, uint16_t *out_payload, uint32_t *out_n,
                                       bm25x_search_stats *stats) {
    using clk = std::chrono::steady_clock;
    const char *who = "bm25x_search_candidates";
    const auto t0 = clk::now();
    std::unique_ptr<CandBatch> b;
    int rc = cand_prepare(who, ix, nq, q_off, q_terms, c_off, c_docs, k, &b);
    if (rc != BM25X_OK) return rc;
    if (stats) BM25X_CUDA_TRY(cudaStreamSynchronize(ix->stream));  // so that h2d_ms means what it says
    const auto t1 = clk::now();
    rc = cand_enqueue(b.get());
    if (rc != BM25X_OK) return rc;
    const auto t2 = clk::now();
    BM25X_CUDA_TRY(b->out.copy_to({out_doc, out_score, out_score64, out_payload, out_n}, nq, k, ix->stream));
    BM25X_CUDA_TRY(cudaStreamSynchronize(ix->stream));
    if (stats) {
        memset(stats, 0, sizeof(*stats));
        rc = b->add_stats(stats);
        stats->h2d_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
        stats->d2h_ms = std::chrono::duration<double, std::milli>(clk::now() - t2).count();
    }
    return rc;
}
