// bm25x_shards.cu — search over a document-sharded index (DESIGN §4.7): every shard answers the batch with its own top-k
// (the whole index's ranking restricted to its documents, because it scores with the whole segment's statistics), and
// k_merge_shards merges the shard lists on shard 0's device into exactly the rows bm25x_search_batch returns on the
// unsharded index.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <vector>

#include "bm25x_common.h"

namespace {

// Row r of shard s: (score64 x, global doc = local + base[s]).  Its rank in the merged list is r plus, for every other
// shard s', the rows of s' ranked before it: score64 >= x for s' < s (equal scores: lower doc ranges first), score64 > x
// for s' > s.  Every row ranks itself — no sort, no shared state; the ranks of the Σ n_s rows are a permutation.
struct ShardRows {
    const uint32_t *doc[BM25X_MAX_SHARDS];
    const float *score[BM25X_MAX_SHARDS];
    const double *score64[BM25X_MAX_SHARDS];
    const uint16_t *payload[BM25X_MAX_SHARDS];
    const uint32_t *n[BM25X_MAX_SHARDS];
    uint32_t base[BM25X_MAX_SHARDS];
};

// rows of a descending list that come before x: score > x (strict) or score >= x (!strict)
__device__ __forceinline__ uint32_t count_before(const double *__restrict__ rows, uint32_t n, double x, bool strict) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const double v = rows[mid];
        if (strict ? v > x : v >= x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// One thread per (query, shard, row slot); consecutive threads take consecutive rows of one shard.  Threads of shard 0 also
// write out_n and fill the slots at or past it as bm25x_batch_prepare leaves them (doc 0xFFFFFFFF, zero scores, payload).
__global__ void k_merge_shards(ShardRows in, uint32_t S, uint32_t nq, uint32_t k, uint32_t *__restrict__ out_doc,
                               float *__restrict__ out_score, double *__restrict__ out_score64,
                               uint16_t *__restrict__ out_payload, uint32_t *__restrict__ out_n) {
    const uint64_t total = (uint64_t)nq * S * k, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const uint32_t r = (uint32_t)(i % k);
        const uint64_t qs = i / k;
        const uint32_t s = (uint32_t)(qs % S), q = (uint32_t)(qs / S);
        const size_t row0 = (size_t)q * k;
        const uint32_t ns = min(in.n[s][q], k);
        if (r < ns) {
            const double x = in.score64[s][row0 + r];
            uint64_t pos = r;
            for (uint32_t t = 0; t < S && pos < k; t++)
                if (t != s) pos += count_before(in.score64[t] + row0, min(in.n[t][q], k), x, t > s);
            if (pos < k) {
                const size_t o = row0 + pos, src = row0 + r;
                out_doc[o] = in.doc[s][src] + in.base[s];
                out_score[o] = in.score[s][src];
                out_score64[o] = x;
                out_payload[o * 3 + 0] = in.payload[s][src * 3 + 0];
                out_payload[o * 3 + 1] = in.payload[s][src * 3 + 1];
                out_payload[o * 3 + 2] = in.payload[s][src * 3 + 2];
            }
        }
        if (s == 0) {
            uint64_t sum = 0;
            for (uint32_t t = 0; t < S; t++) sum += min(in.n[t][q], k);
            const uint32_t nout = sum < k ? (uint32_t)sum : k;
            if (r == 0) out_n[q] = nout;
            if (r >= nout) {
                const size_t o = row0 + r;
                out_doc[o] = BM25X_DOC_INF;
                out_score[o] = 0.f;
                out_score64[o] = 0.0;
                out_payload[o * 3 + 0] = out_payload[o * 3 + 1] = out_payload[o * 3 + 2] = 0;
            }
        }
    }
}

int launch_merge(int device, const ShardRows &in, uint32_t S, uint32_t nq, uint32_t k, const ResultRows &out,
                 cudaStream_t st) {
    const uint64_t total = (uint64_t)nq * S * k;
    if (!total) return BM25X_OK;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    const uint64_t want = (total + 255) / 256, cap = (uint64_t)sms * 32;
    k_merge_shards<<<(unsigned)std::min(want, cap), 256, 0, st>>>(in, S, nq, k, out.doc, out.score, out.score64,
                                                                  out.payload, out.n);
    BM25X_CUDA_TRY(cudaGetLastError());
    return BM25X_OK;
}

void set_shard(ShardRows &in, uint32_t s, const ResultRows &rows, uint32_t base) {
    in.doc[s] = rows.doc;
    in.score[s] = rows.score;
    in.score64[s] = rows.score64;
    in.payload[s] = rows.payload;
    in.n[s] = rows.n;
    in.base[s] = base;
}

// Bits [lo, hi) of a bitmap over global doc ids, shifted to bit 0 (shard bounds need not be multiples of 8).
std::vector<uint8_t> allow_slice(const uint8_t *allow, uint32_t n_docs, uint32_t lo, uint32_t hi) {
    const size_t nb = ((size_t)(hi - lo) + 7) / 8, total = ((size_t)n_docs + 7) / 8;
    std::vector<uint8_t> out(nb ? nb : 1, 0);
    const size_t byte0 = lo >> 3;
    const unsigned sh = lo & 7u;
    for (size_t j = 0; j < nb; j++) {
        unsigned v = allow[byte0 + j] >> sh;
        if (sh && byte0 + j + 1 < total) v |= (unsigned)allow[byte0 + j + 1] << (8 - sh);
        out[j] = (uint8_t)v;
    }
    if ((hi - lo) & 7u) out[nb - 1] &= (uint8_t)((1u << ((hi - lo) & 7u)) - 1u);  // no bits past the shard's last doc
    return out;
}

}  // namespace

extern "C" int bm25x_sharded_search_batch(bm25x_sharded_index *sx, uint32_t nq, const uint32_t *q_off,
                                          const uint32_t *q_terms, uint32_t k, const uint8_t *allow, uint32_t *out_doc,
                                          float *out_score, double *out_score64, uint16_t *out_payload, uint32_t *out_n,
                                          bm25x_search_stats *stats) {
    using clk = std::chrono::steady_clock;
    if (!sx) {
        bm25x_set_error("bm25x_sharded_search_batch: null argument");
        return BM25X_ERR_INVALID;
    }
    const auto t0 = clk::now();
    // ---- the refusals of bm25x_search_batch: its argument checks, then its canonicalisation slice by slice against the
    // WHOLE segment's df (a query with 65 live terms is refused even when no shard sees more than 64) ----
    if (nq && (!q_off || (!q_terms && q_off[nq] != 0))) {
        bm25x_set_error("bm25x_batch_prepare: null argument");
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
    uint32_t n_live = 0;  // live queries of the whole index
    int rc = BM25X_OK;
    {
        const SlicePlan plan(sx->shards[0]->slice_min, nq);
        CanonQueries cq;
        for (uint32_t s = 0; s < plan.n && rc == BM25X_OK; s++) {
            const uint32_t a = plan.begin(s), e = plan.begin(s + 1);
            rc = bm25x_canonicalise(sx->h_df.data(), sx->n_terms, e - a, q_off + a, q_terms, &cq);
            for (uint32_t i = 0; i < e - a; i++) n_live += cq.live[i] != 0;
        }
    }
    if (rc != BM25X_OK) return rc;
    const uint32_t S = sx->n_shards;
    bm25x_index *ix0 = sx->shards[0];
    const int dev0 = ix0->device;
    cudaStream_t ms = ix0->stream;  // the merge runs behind shard 0's kernels on its library stream
    std::vector<bm25x_batch *> bs(S, nullptr);
    std::vector<ResultRows> peer(S);  // rows of shards on other devices, copied to dev0
    std::vector<cudaEvent_t> evs;
    ResultRows mo;
    auto cleanup = [&](int code) {
        cudaSetDevice(dev0);
        cudaStreamSynchronize(ms);
        for (ResultRows &p : peer) p.release(ms);
        mo.release(ms);
        for (cudaEvent_t e : evs) cudaEventDestroy(e);
        for (bm25x_batch *b : bs)
            if (b) bm25x_batch_destroy(b);
        return code;
    };
    // ---- prepare + run shard after shard: the next shard's canonicalisation overlaps the kernels of the previous ----
    for (uint32_t s = 0; s < S && rc == BM25X_OK; s++) {
        const uint32_t lo = sx->bounds[s], hi = sx->bounds[s + 1];
        std::vector<uint8_t> al;
        if (allow) al = allow_slice(allow, sx->n_docs, lo, hi);
        rc = bm25x_batch_prepare(sx->shards[s], nq, q_off, q_terms, k, allow ? al.data() : nullptr, &bs[s]);
        if (rc == BM25X_OK) rc = bm25x_batch_run_timed(bs[s]);
    }
    if (rc != BM25X_OK) return cleanup(rc);
    const auto t1 = clk::now();
    // ---- shard rows on dev0: read in place there, copied peer to peer from the other devices ----
    ShardRows in;
    memset(&in, 0, sizeof(in));
    cudaError_t e = cudaSetDevice(dev0);
    for (uint32_t s = 0; s < S && e == cudaSuccess; s++) {
        e = cudaStreamWaitEvent(ms, bm25x_batch_done_event(bs[s]), 0);
        const ResultRows *rows = &bm25x_batch_rows(bs[s]);
        if (e == cudaSuccess && sx->shards[s]->device != dev0) {
            e = peer[s].alloc(nq, k, ms);
            if (e == cudaSuccess) e = rows->copy_to(peer[s], nq, k, ms);
            rows = &peer[s];
        }
        set_shard(in, s, *rows, sx->bounds[s]);
    }
    if (e == cudaSuccess) e = mo.alloc(nq, k, ms);
    cudaEvent_t m0 = nullptr, m1 = nullptr;
    if (e == cudaSuccess && stats) {
        e = cudaEventCreate(&m0);
        if (e == cudaSuccess) evs.push_back(m0);
        if (e == cudaSuccess) e = cudaEventCreate(&m1);
        if (e == cudaSuccess) evs.push_back(m1);
        if (e == cudaSuccess) e = cudaEventRecord(m0, ms);
    }
    if (e != cudaSuccess) {
        bm25x_set_error("bm25x_sharded_search_batch: %s", cudaGetErrorString(e));
        return cleanup(e == cudaErrorMemoryAllocation ? BM25X_ERR_OOM : BM25X_ERR_CUDA);
    }
    rc = launch_merge(dev0, in, S, nq, k, mo, ms);
    if (rc != BM25X_OK) return cleanup(rc);
    if (stats) e = cudaEventRecord(m1, ms);
    if (e == cudaSuccess) e = mo.copy_to({out_doc, out_score, out_score64, out_payload, out_n}, nq, k, ms);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ms);  // after the merge: every shard's kernels have finished too
    if (e != cudaSuccess) {
        bm25x_set_error("bm25x_sharded_search_batch: %s", cudaGetErrorString(e));
        return cleanup(BM25X_ERR_CUDA);
    }
    if (stats) {
        memset(stats, 0, sizeof(*stats));
        for (uint32_t s = 0; s < S && rc == BM25X_OK; s++) rc = bm25x_batch_add_stats(bs[s], stats);
        float mms = 0.f;
        if (rc == BM25X_OK) {
            cudaSetDevice(dev0);
            e = cudaEventElapsedTime(&mms, m0, m1);
            if (e != cudaSuccess) {
                bm25x_set_error("bm25x_sharded_search_batch: %s", cudaGetErrorString(e));
                rc = BM25X_ERR_CUDA;
            }
        }
        stats->kernel_ms += mms;  // summed device time of the shards' kernels and the merge, not wall time
        stats->launches += (uint64_t)nq * S * k ? 1u : 0u;
        stats->queries = n_live;
        stats->h2d_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
        stats->d2h_ms = std::chrono::duration<double, std::milli>(clk::now() - t1).count();
    }
    return cleanup(rc);
}

// ---- test / measurement hook: the merge kernel alone on host rows ----
extern "C" int bm25x_merge_shards(int device, uint32_t S, uint32_t nq, uint32_t k, const uint32_t *doc_base,
                                  const uint32_t *doc, const float *score, const double *score64, const uint16_t *payload,
                                  const uint32_t *n, uint32_t *out_doc, float *out_score, double *out_score64,
                                  uint16_t *out_payload, uint32_t *out_n, float *merge_ms) {
    const char *who = "bm25x_merge_shards";
    if (k == 0) {
        bm25x_set_error("number of needed rows is set to 0");
        return BM25X_ERR_LIMIT_ZERO;
    }
    if (S == 0 || S > BM25X_MAX_SHARDS || k > BM25X_MAX_K) {
        bm25x_set_error("%s: n_shards=%u must be 1..%d and k=%u <= %d", who, S, BM25X_MAX_SHARDS, k, BM25X_MAX_K);
        return BM25X_ERR_INVALID;
    }
    if (nq && (!doc_base || !doc || !score || !score64 || !payload || !n)) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        bm25x_set_error("%s: CUDA device %d not available (%d devices); there is no CPU fallback", who, device, ndev);
        return BM25X_ERR_CUDA;
    }
    BM25X_CUDA_TRY(cudaSetDevice(device));
    cudaStream_t st = nullptr;
    BM25X_CUDA_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    // the S shards' rows back to back: S * nq rows, on the host and in `src`
    const ResultRows host{const_cast<uint32_t *>(doc), const_cast<float *>(score), const_cast<double *>(score64),
                          const_cast<uint16_t *>(payload), const_cast<uint32_t *>(n)};
    ResultRows src, mo;
    cudaEvent_t m0 = nullptr, m1 = nullptr;
    cudaError_t e = src.alloc((size_t)nq * S, k, st);
    if (e == cudaSuccess) e = mo.alloc(nq, k, st);
    if (e == cudaSuccess) e = host.copy_to(src, (size_t)nq * S, k, st);
    ShardRows in;
    memset(&in, 0, sizeof(in));
    for (uint32_t s = 0; s < S; s++) set_shard(in, s, src.from((size_t)s * nq, k), nq ? doc_base[s] : 0);
    if (e == cudaSuccess) e = cudaEventCreate(&m0);
    if (e == cudaSuccess) e = cudaEventCreate(&m1);
    if (e == cudaSuccess) e = cudaEventRecord(m0, st);
    int rc = BM25X_OK;
    if (e == cudaSuccess) rc = launch_merge(device, in, S, nq, k, mo, st);
    if (e == cudaSuccess && rc == BM25X_OK) e = cudaEventRecord(m1, st);
    if (e == cudaSuccess && rc == BM25X_OK) e = mo.copy_to({out_doc, out_score, out_score64, out_payload, out_n}, nq, k, st);
    if (e == cudaSuccess && rc == BM25X_OK) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess && rc == BM25X_OK && merge_ms) e = cudaEventElapsedTime(merge_ms, m0, m1);
    cudaStreamSynchronize(st);
    src.release(st);
    mo.release(st);
    cudaStreamSynchronize(st);
    if (m0) cudaEventDestroy(m0);
    if (m1) cudaEventDestroy(m1);
    cudaStreamDestroy(st);
    if (rc != BM25X_OK) return rc;
    if (e != cudaSuccess) {
        bm25x_set_error("%s: %s", who, cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? BM25X_ERR_OOM : BM25X_ERR_CUDA;
    }
    return BM25X_OK;
}

// ---- handle queries and options ----
extern "C" int bm25x_sharded_get_info(const bm25x_sharded_index *sx, bm25x_index_info *out, uint32_t *n_shards_out,
                                      uint32_t *doc_bounds_out) {
    if (!sx || !out) {
        bm25x_set_error("bm25x_sharded_get_info: null argument");
        return BM25X_ERR_INVALID;
    }
    memset(out, 0, sizeof(*out));
    out->n_docs = sx->n_docs;
    out->n_terms = sx->n_terms;
    out->n_postings = sx->n_post;
    out->sum_doc_len = sx->sum_len;
    out->avgdl = sx->avgdl;
    out->k1 = sx->k1;
    out->b = sx->b;
    for (const bm25x_index *ix : sx->shards) {
        out->device_bytes += ix->device_bytes;
        out->n_blocks += ix->d.n_blocks;
    }
    out->device = sx->shards[0]->device;
    if (n_shards_out) *n_shards_out = sx->n_shards;
    if (doc_bounds_out) std::copy(sx->bounds.begin(), sx->bounds.end(), doc_bounds_out);
    return BM25X_OK;
}

extern "C" int bm25x_sharded_get_shard(const bm25x_sharded_index *sx, uint32_t s, bm25x_index_layout *layout,
                                       bm25x_index_derived *derived) {
    if (!sx) {
        bm25x_set_error("bm25x_sharded_get_shard: null argument");
        return BM25X_ERR_INVALID;
    }
    if (s >= sx->n_shards) {
        bm25x_set_error("bm25x_sharded_get_shard: shard %u of %u", s, sx->n_shards);
        return BM25X_ERR_INVALID;
    }
    int rc = layout ? bm25x_index_get_layout(sx->shards[s], layout) : BM25X_OK;
    if (rc == BM25X_OK && derived) rc = bm25x_index_get_derived(sx->shards[s], derived);
    return rc;
}

extern "C" int bm25x_sharded_set_option(bm25x_sharded_index *sx, const char *name, int64_t value) {
    if (!sx || !name) {
        bm25x_set_error("bm25x_sharded_set_option: null argument");
        return BM25X_ERR_INVALID;
    }
    for (bm25x_index *ix : sx->shards) {
        const int rc = bm25x_index_set_option(ix, name, value);
        if (rc != BM25X_OK) return rc;  // an unknown name fails on shard 0, before any shard changed
    }
    return BM25X_OK;
}

// Every shard knows every term (ordinals are the segment's); shard 0 holds the keys.
extern "C" int bm25x_sharded_lookup_terms(const bm25x_sharded_index *sx, const uint8_t *keys, uint32_t n, uint32_t *out) {
    return bm25x_lookup_terms(sx ? sx->shards[0] : nullptr, keys, n, out);
}
