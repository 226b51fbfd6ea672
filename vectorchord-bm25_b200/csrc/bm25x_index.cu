// bm25x_index.cu — index lifetime: host CSR (the reference's sealed Segment) → flat HBM layout.
//
// Replaces, for the read path, bm25::build → flush (crates/bm25/src/build.rs:22-71,
// crates/bm25/src/flush.rs:40-158): same semantics (N, Σlen → avgdl from exact lengths, per-document
// quantised fieldnorm, 128-posting blocks in (term, doc) order with min/max doc per block, df per
// token) but none of its page / tape / address-tree machinery.  Layout in DESIGN.md §3.
#include <math.h>
#include <omp.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <optional>

#include "bm25x_common.h"
#include "bm25x_blocks.cuh"

static thread_local char g_err[512] = "";

void bm25x_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char *bm25x_last_error(void) { return g_err; }

int bm25x_host_threads(int cap) {
    static const int granted = [] {
        if (const char *e = getenv("BM25X_HOST_THREADS")) {  // explicit share, e.g. cores / ranks when several ranks share a box
            const int v = atoi(e);
            if (v >= 1) return v;
        }
        int n = omp_get_num_procs();  // honours the affinity mask
        FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
        if (f) {
            char q[64];
            long long per = 0;
            if (fscanf(f, "%63s %lld", q, &per) == 2 && strcmp(q, "max") != 0 && per > 0) {
                const long long quota = (atoll(q) + per / 2) / per;
                if (quota >= 1 && quota < n) n = (int)quota;
            }
            fclose(f);
        } else if ((f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r"))) {
            long long quota = -1, per = 100000;
            if (fscanf(f, "%lld", &quota) != 1) quota = -1;
            fclose(f);
            FILE *g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
            if (g) {
                if (fscanf(g, "%lld", &per) != 1) per = 100000;
                fclose(g);
            }
            if (quota > 0 && per > 0 && (quota + per / 2) / per < n) n = (int)std::max<long long>(1, (quota + per / 2) / per);
        }
        return n < 1 ? 1 : n;
    }();
    return cap > 0 && granted > cap ? cap : granted;
}

extern "C" int bm25x_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

// ---- fieldnorm codec (crates/bm25/src/bm25.rs:15-283): 0..=40 step 1, then groups of 8 whose step
// doubles per group.  Generated, and pinned against the reference's literal table by the tests. ----
static uint32_t g_fn_len[256];
static bool g_fn_ready = false;
static void fn_init() {
    if (g_fn_ready) return;
    int n = 0;
    for (; n <= 40; n++) g_fn_len[n] = (uint32_t)n;
    uint32_t v = 40, step = 2;
    while (n < 256) {
        for (int i = 0; i < 8 && n < 256; i++) {
            v += step;
            g_fn_len[n++] = v;
        }
        step *= 2;
    }
    g_fn_ready = true;
}
uint32_t bm25x_fieldnorm_to_length(uint8_t fn) {
    fn_init();
    return g_fn_len[fn];
}
uint8_t bm25x_length_to_fieldnorm(uint32_t len) {  // bm25.rs:278-283
    fn_init();
    int lo = 0, hi = 256;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (g_fn_len[mid] <= len) lo = mid + 1;
        else hi = mid;
    }
    return (uint8_t)(lo - 1);
}

// Cache::new (bm25.rs:340-354): s0 = idf·(k1 + 1) of a term in n of N documents (bm25.rs:285-289,348), and the s1 table,
// identical for every term: it depends only on (k1, b, avgdl) (bm25.rs:349-352).
static double bm25_s0(double n, double N, double k1) {
    double idf = log((N + 1.0) / (n + 0.5));
    return idf * (k1 + 1.0);
}
static void bm25_s1(double k1, double b, double avgdl, double s1d[256]) {
    fn_init();
    for (int f = 0; f < 256; f++) {
        double dl = (double)g_fn_len[f];
        s1d[f] = k1 * (1.0 - b + b * dl / avgdl);
    }
}

// flush.rs:52-66: the norms of N documents into fn (when not NULL) and their Σlen — quantised from the exact lengths, or,
// without doc_len, as the stored index keeps them: the norm per document and the exact total (tuples.rs:141-160,756-762).
static uint64_t doc_norms(uint32_t N, const uint32_t *doc_len, const uint8_t *stored_fn, uint64_t stored_sum, uint8_t *fn) {
    fn_init();
    if (!doc_len) {
        if (fn) memcpy(fn, stored_fn, N);
        return stored_sum;
    }
    uint64_t sum_len = 0;
#pragma omp parallel for reduction(+ : sum_len) num_threads(bm25x_host_threads(0))
    for (uint32_t d = 0; d < N; d++) {
        sum_len += doc_len[d];
        if (fn) fn[d] = bm25x_length_to_fieldnorm(doc_len[d]);
    }
    return sum_len;
}

// The statistics a handle scores with: avgdl and the s0 / s1 tables of a segment of N documents with the given df.  The
// only place they are computed: the shards of a segment and its growing segment receive the segment's object, so that
// they score with its bits (DESIGN §4.7).
struct Stats {
    uint64_t sum_len;
    double avgdl;
    std::vector<double> s0d;  // [T]
    std::vector<float> s0f;
    double s1d[256];
    float s1f[256];

    Stats(uint32_t N, uint64_t sum_len, double avgdl, const uint32_t *df, uint32_t T, double k1, double b)
        : sum_len(sum_len), avgdl(avgdl), s0d(T), s0f(T) {
        for (uint32_t t = 0; t < T; t++) {
            s0d[t] = bm25_s0((double)df[t], (double)N, k1);
            s0f[t] = (float)s0d[t];
        }
        bm25_s1(k1, b, avgdl, s1d);
        for (int f = 0; f < 256; f++) s1f[f] = (float)s1d[f];
    }
    // a segment's own: avgdl = Σlen / N (flush.rs:52-66)
    Stats(uint32_t N, uint64_t sum_len, const uint32_t *df, uint32_t T, double k1, double b)
        : Stats(N, sum_len, (double)sum_len / (double)N, df, T, k1, b) {}
};

// Smallest s1 over the norms of the documents present: the one-compare single-term test of k_search_ring needs a lower
// bound.
static float s1f_min(const uint8_t *fn, uint32_t N, const float s1f[256]) {
    bool seen[256] = {false};
    for (uint32_t d = 0; d < N; d++) seen[fn[d]] = true;
    float mn = 3.0e38f;
    for (int f = 0; f < 256; f++)
        if (seen[f] && s1f[f] < mn) mn = s1f[f];
    return mn;
}

// ---- device transforms ----

// CSR chunk → AoS postings at their padded positions, with the fieldnorm byte folded in.
__global__ void k_build_postings(const uint32_t *__restrict__ c_doc, const uint32_t *__restrict__ c_tf,
                                 uint64_t chunk_base, uint64_t chunk_n, const uint64_t *__restrict__ off,
                                 const uint64_t *__restrict__ off_pad, uint32_t n_terms,
                                 const uint8_t *__restrict__ fieldnorm, Posting *__restrict__ post) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= chunk_n) return;
    uint64_t gi = chunk_base + i;
    const uint32_t t = owner_of(off, n_terms, gi);
    uint32_t d = c_doc[i];
    Posting p;
    p.doc = d;
    p.w = (c_tf[i] << 8) | fieldnorm[d];
    post[off_pad[t] + (gi - off[t])] = p;
}

__global__ void k_pad_slots(const uint64_t *__restrict__ off_pad, const uint32_t *__restrict__ df, uint32_t n_terms,
                            Posting *__restrict__ post) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_terms) return;
    Posting p;
    p.doc = BM25X_DOC_INF;
    p.w = 0;
    const uint32_t end = (df[t] + BM25X_POST_ALIGN - 1u) & ~(BM25X_POST_ALIGN - 1u);
    for (uint32_t i = df[t]; i < end; i++) post[off_pad[t] + i] = p;
}

// pdoc[i] = post[i].doc: the doc-id-only copy streamed by the 2..4-term classes of k_search_ring (bm25x_search_ring.cuh,
// RCfg::DOCRING).  Derived data: built here for every way an index comes to life (postings, stored blocks, replica).
__global__ void k_extract_docs(const Posting *__restrict__ post, uint64_t n, uint32_t *__restrict__ pdoc) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) pdoc[i] = post[i].doc;
}

// Per 128-posting block: (first doc, last doc) = SummaryTuple.{min,max}_document_id, and the block's score bound =
// Cache::evaluate of the block's arg-max posting, what the reference keeps as SummaryTuple.(wand_fieldnorm,
// wand_term_frequency) (flush.rs:101-120) and evaluates per block at query time (search.rs:381,426-429).  Stored as f32
// rounded UP after the same 2^-40 inflation as the token-level bound (block_bound).
__global__ void k_block_desc(const uint64_t *__restrict__ off_pad, const uint32_t *__restrict__ df,
                             const uint64_t *__restrict__ blk_off, uint32_t n_terms, uint64_t n_blocks,
                             const Posting *__restrict__ post, const double *__restrict__ s0d,
                             const double *__restrict__ s1d, uint2 *__restrict__ blk, float *__restrict__ blk_ub) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_blocks) return;
    const uint32_t t = owner_of(blk_off, n_terms, g);
    uint64_t first = (g - blk_off[t]) * BM25X_BLOCK;
    uint64_t last = first + BM25X_BLOCK;
    if (last > df[t]) last = df[t];
    blk[g] = make_uint2(post[off_pad[t] + first].doc, post[off_pad[t] + last - 1].doc);
    const double s0 = s0d[t];
    double best = 0.0;
    for (uint64_t i = first; i < last; i++) {
        const double v = posting_score(post[off_pad[t] + i].w, s0, s1d);
        best = v > best ? v : best;
    }
    blk_ub[g] = block_bound(best);
}

// Ingest check: the stored SummaryTuple.(wand_fieldnorm, wand_term_frequency) of a block must evaluate to the block's
// real maximum (it is the arg-max of the block's own postings, flush.rs:101-110); anything else is a corrupt index.
__global__ void k_check_block_wand(uint64_t n_blocks, const uint64_t *__restrict__ blk_off, uint32_t n_terms,
                                   const uint8_t *__restrict__ wand_fn, const uint32_t *__restrict__ wand_tf,
                                   const double *__restrict__ s0d, const double *__restrict__ s1d,
                                   const float *__restrict__ blk_ub, uint32_t *__restrict__ err) {
    uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_blocks) return;
    const uint32_t t = owner_of(blk_off, n_terms, g);
    if (!wand_pair_ok(wand_tf[g], wand_fn[g], s0d[t], s1d, blk_ub[g])) atomicOr(err, BM25X_BLKERR_WAND);
}

// Per-term upper bound of a single posting's exact score: max over the term's postings of Cache::evaluate
// (bm25.rs:355-358) — what the reference stores as the token-level (wand_fieldnorm, wand_term_frequency) arg-max
// (flush.rs:101-120) and evaluates at query time (search.rs:363).  One block per term; inflated by UB_INFLATE, in f64.
__global__ void k_term_ub(const uint64_t *__restrict__ off_pad, const uint32_t *__restrict__ df,
                          const Posting *__restrict__ post, const double *__restrict__ s0d,
                          const double *__restrict__ s1d, uint32_t n_terms, double *__restrict__ ubd) {
    __shared__ double red[256];
    for (uint32_t t = blockIdx.x; t < n_terms; t += gridDim.x) {
        const Posting *pp = post + off_pad[t];
        const double s0 = s0d[t];
        double best = 0.0;
        for (uint32_t i = threadIdx.x; i < df[t]; i += blockDim.x) {
            const double v = posting_score(pp[i].w, s0, s1d);
            best = v > best ? v : best;
        }
        red[threadIdx.x] = best;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if ((int)threadIdx.x < o && red[threadIdx.x + o] > red[threadIdx.x]) red[threadIdx.x] = red[threadIdx.x + o];
            __syncthreads();
        }
        if (threadIdx.x == 0) ubd[t] = red[0] * UB_INFLATE;
        __syncthreads();
    }
}

// Champion lists: one warp per term keeps the best L postings by (exact single-term score desc, doc id asc) — the order in
// which single-term documents enter a result (Cache::evaluate, bm25.rs:355-358, is the whole score of such a document).
// The list is scanned once in doc order; a posting is buffered only if it beats the current L-th best (later documents
// lose ties), and the 2L-entry buffer is sorted and cut back to L when it fills.
#define CHAMP_WARPS 4
__global__ void __launch_bounds__(CHAMP_WARPS * 32) k_champions(const uint64_t *__restrict__ off_pad, const uint32_t *__restrict__ df,
                                                                const Posting *__restrict__ post, const double *__restrict__ s0d,
                                                                const double *__restrict__ s1d, uint32_t n_terms,
                                                                const uint64_t *__restrict__ champ_off, Posting *__restrict__ champ) {
    constexpr int L = (int)BM25X_CHAMP_L, CAP = 2 * L;
    __shared__ double bs[CHAMP_WARPS][CAP];
    __shared__ uint32_t bd[CHAMP_WARPS][CAP], bw[CHAMP_WARPS][CAP];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double *ss = bs[wid];
    uint32_t *sd = bd[wid], *sw = bw[wid];
    const uint32_t lt = (1u << lane) - 1u;
    auto sort_buf = [&](int n) {  // bitonic over CAP entries, best first; entries >= n are padding (score -1)
        for (int i = n + lane; i < CAP; i += 32) {
            ss[i] = -1.0;
            sd[i] = BM25X_DOC_INF;
            sw[i] = 0;
        }
        __syncwarp();
        for (int size = 2; size <= CAP; size <<= 1)
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int i = lane; i < CAP / 2; i += 32) {
                    const int a = 2 * i - (i & (stride - 1)), b = a + stride;
                    const double sa = ss[a], sb = ss[b];
                    const uint32_t da = sd[a], db = sd[b];
                    const bool a_first = sa > sb || (sa == sb && da < db);
                    const bool desc = (a & size) == 0;
                    if (desc ? !a_first : a_first) {
                        ss[a] = sb;
                        ss[b] = sa;
                        sd[a] = db;
                        sd[b] = da;
                        const uint32_t t = sw[a];
                        sw[a] = sw[b];
                        sw[b] = t;
                    }
                }
                __syncwarp();
            }
    };
    for (uint32_t t = blockIdx.x * CHAMP_WARPS + wid; t < n_terms; t += gridDim.x * CHAMP_WARPS) {
        const Posting *pp = post + off_pad[t];
        const uint32_t n = df[t];
        const double s0 = s0d[t];
        int cnt = 0;
        bool have = false;
        double thr = 0.0;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane;
            Posting v;
            v.doc = 0;
            v.w = 0;
            double sc = -1.0;
            if (i < n) {
                v = pp[i];
                sc = posting_score(v.w, s0, s1d);
            }
            const bool acc = i < n && (!have || sc > thr);
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, acc);
            if (acc) {
                const int at = cnt + __popc(m & lt);
                ss[at] = sc;
                sd[at] = v.doc;
                sw[at] = v.w;
            }
            cnt += __popc(m);
            if (cnt > CAP - 32) {
                __syncwarp();
                sort_buf(cnt);
                cnt = L;
                thr = ss[L - 1];
                have = true;
                __syncwarp();
            }
        }
        __syncwarp();
        sort_buf(cnt);
        const int keep = cnt < L ? cnt : L;
        Posting *out = champ + champ_off[t];
        for (int i = lane; i < keep; i += 32) {
            Posting v;
            v.doc = sd[i];
            v.w = sw[i];
            out[i] = v;
        }
        __syncwarp();
    }
}

template <typename T>
static int dev_alloc(bm25x_index *ix, T **p, size_t n) {
    size_t bytes = sizeof(T) * (n ? n : 1);
    BM25X_CUDA_TRY(cudaMalloc((void **)p, bytes));
    ix->allocs.push_back((void *)*p);
    ix->device_bytes += bytes;
    return BM25X_OK;
}

// The arrays of a handle, sized by the counts in ix->d: index_begin fills them, a replica receives them.
static int alloc_arrays(bm25x_index *ix) {
    DeviceIndex &d = ix->d;
    const size_t T = d.n_terms, N = d.n_docs, PP = d.n_post_pad + BM25X_POST_SLACK;
    int rc = BM25X_OK;
    auto a = [&](auto **p, size_t n) {
        if (rc == BM25X_OK) rc = dev_alloc(ix, p, n);
    };
    a(&d.post, PP);
    a(&d.pdoc, PP);
    a(&d.post_off, T + 1);
    a(&d.df, T);
    a(&d.blk_off, T + 1);
    a(&d.blk, d.n_blocks);
    a(&d.blk_ub, d.n_blocks);
    a(&d.s0f, T);
    a(&d.s0d, T);
    a(&d.s1d, 256);
    a(&d.s1f, 256);
    a(&d.ubd, T);
    a(&d.fieldnorm, N);
    a(&d.payload, N * 3);
    return rc;
}

// champ_off from the host copy of df, then the lists (index_finish_device / finalize_replica; needs post, s0d, s1d).
// Called again for a replica that is refilled and finalized once more: the lists are rebuilt from the new postings, in the
// same allocation when their total length has not changed.
static cudaError_t build_champions(bm25x_index *ix) {
    DeviceIndex &d = ix->d;
    const uint32_t T = d.n_terms;
    std::vector<uint64_t> h_off((size_t)T + 1);
    uint64_t run = 0;
    for (uint32_t t = 0; t < T; t++) {
        h_off[t] = run;
        run += std::min<uint32_t>(ix->h_df[t], BM25X_CHAMP_L);
    }
    h_off[T] = run;
    cudaError_t e = cudaSuccess;
    if (d.champ && run != d.n_champ) {
        cudaFree(d.champ);
        ix->allocs.erase(std::find(ix->allocs.begin(), ix->allocs.end(), (void *)d.champ));
        ix->device_bytes -= sizeof(Posting) * (size_t)(d.n_champ ? d.n_champ : 1);
        d.champ = nullptr;
    }
    d.n_champ = run;
    if (!d.champ) {
        e = cudaMalloc((void **)&d.champ, sizeof(Posting) * (size_t)(run ? run : 1));
        if (e != cudaSuccess) {
            d.champ = nullptr;
            return e;
        }
        ix->allocs.push_back((void *)d.champ);
        ix->device_bytes += sizeof(Posting) * (size_t)(run ? run : 1);
    }
    if (!d.champ_off) {  // n_terms + 1 entries: the size never changes
        e = cudaMalloc((void **)&d.champ_off, sizeof(uint64_t) * ((size_t)T + 1));
        if (e != cudaSuccess) {
            d.champ_off = nullptr;
            return e;
        }
        ix->allocs.push_back((void *)d.champ_off);
        ix->device_bytes += sizeof(uint64_t) * ((size_t)T + 1);
    }
    e = cudaMemcpy(d.champ_off, h_off.data(), sizeof(uint64_t) * ((size_t)T + 1), cudaMemcpyHostToDevice);
    if (e != cudaSuccess || !T) return e;
    const unsigned blocks = (unsigned)std::min<uint64_t>(((uint64_t)T + CHAMP_WARPS - 1) / CHAMP_WARPS, (uint64_t)ix->sm_count * 16ull);
    k_champions<<<blocks, CHAMP_WARPS * 32>>>(d.post_off, d.df, d.post, d.s0d, d.s1d, T, d.champ_off, d.champ);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return e;
}

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
};

// The refusal for a failed CUDA call of a build step.
static int cuda_refusal(const char *who, const char *step, cudaError_t e) {
    bm25x_set_error("%s: %s failed: %s", who, step, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? BM25X_ERR_OOM : BM25X_ERR_CUDA;
}

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

static int check_device(const char *who, int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        bm25x_set_error("%s: CUDA device %d not available (%d devices); there is no CPU fallback", who, device, ndev);
        return BM25X_ERR_CUDA;
    }
    return BM25X_OK;
}

static int check_common(const char *who, uint32_t n_docs, const void *doc_len, double k1, double b, int device) {
    if (n_docs == 0 || n_docs == BM25X_DOC_INF || !doc_len) {
        bm25x_set_error("%s: empty or malformed corpus", who);
        return BM25X_ERR_INVALID;
    }
    if (!(k1 >= 0.0) || !(b >= 0.0 && b <= 1.0)) {
        bm25x_set_error("%s: k1/b out of range", who);
        return BM25X_ERR_INVALID;
    }
    return check_device(who, device);
}

static int check_keys(const char *who, const uint8_t *term_key, uint32_t T) {
    if (term_key)
        for (uint32_t t = 1; t < T; t++)
            if (memcmp(term_key + (size_t)(t - 1) * 16, term_key + (size_t)t * 16, 16) >= 0) {
                bm25x_set_error("%s: term_key must be strictly ascending", who);
                return BM25X_ERR_INVALID;
            }
    return BM25X_OK;
}

// Environment overrides of the option defaults (test matrix: BM25X_SEED=0 / BM25X_TWOPHASE=1 run the same tests through
// the other kernel paths); bm25x_index_set_option still wins.
static void apply_env_options(bm25x_index *ix) {
    if (const char *e = getenv("BM25X_SEED")) ix->seed = atoi(e) != 0;
    if (const char *e = getenv("BM25X_TWOPHASE")) ix->twophase = atoi(e) != 0;
    if (const char *e = getenv("BM25X_SEED_FORCE")) {  // every eligible query through the seeded kernel, dense or skewed
        if (atoi(e) != 0) {
            ix->seed_prune_min = 0xFFFFFFFFu;
            ix->seed_dense_div = 0u;
        }
    }
}

// A new handle on `device`: checked to be sm_90, its streams created, the pool kept, the options' defaults set.  `who`
// names the entry point in the refusal.
static int handle_open(const char *who, int device, IndexGuard &ix) {
    ix.reset(new bm25x_index());
    apply_env_options(ix.get());
    ix->device = device;
    BM25X_CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    BM25X_CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        bm25x_set_error("%s: device %d is sm_%d%d; this library only carries sm_90a kernels", who, device, prop.major,
                        prop.minor);
        return BM25X_ERR_CUDA;
    }
    ix->sm_count = prop.multiProcessorCount;
    BM25X_CUDA_TRY(cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking));
    // created with the handle, never later: concurrent first calls of bm25x_search_batch must not race to create it
    BM25X_CUDA_TRY(cudaStreamCreateWithFlags(&ix->copy_stream, cudaStreamNonBlocking));
    {   // keep freed batch buffers cached in the default pool (bm25x_batch_* allocate stream-ordered)
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
            uint64_t thr = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
    }
    return BM25X_OK;
}

// A handle with everything but the postings, scoring with the `given` statistics (a shard's or a growing segment's: its
// segment's) or, when NULL, its own.  Refusals name bm25x_index_create whichever entry point builds.
static int index_begin(const BuildMeta &m, const Stats *given, int device, IndexGuard &ix) {
    int rc = handle_open("bm25x_index_create", device, ix);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = m.n_docs, T = m.n_terms;
    ix->k1 = m.k1;
    ix->b = m.b;
    std::vector<uint8_t> h_fn(N);
    ix->sum_len = doc_norms(N, m.doc_len, m.fieldnorm, m.sum_len, h_fn.data());
    std::optional<Stats> own;
    const Stats &st = given ? *given : own.emplace(N, ix->sum_len, m.df, T, m.k1, m.b);
    ix->avgdl = st.avgdl;
    ix->s1f_min = s1f_min(h_fn.data(), N, st.s1f);

    // ---- per-term df, padded offsets, block offsets ----
    ix->h_df.assign(m.df, m.df + T);
    std::vector<uint64_t> h_off_pad(T + 1), h_blk_off(T + 1);
    uint64_t pp = 0, nb = 0;
    for (uint32_t t = 0; t < T; t++) {
        const uint64_t n = m.df[t];
        h_off_pad[t] = pp;
        h_blk_off[t] = nb;
        pp += (n + BM25X_POST_ALIGN - 1) & ~(uint64_t)(BM25X_POST_ALIGN - 1);
        nb += (n + BM25X_BLOCK - 1) / BM25X_BLOCK;
    }
    h_off_pad[T] = pp;
    h_blk_off[T] = nb;
    if (m.term_key) ix->h_keys.assign(m.term_key, m.term_key + (size_t)T * 16);

    DeviceIndex &d = ix->d;
    d.n_docs = N;
    d.n_terms = T;
    d.n_post = m.n_post;
    d.n_post_pad = pp;
    d.n_blocks = nb;
    rc = alloc_arrays(ix.get());
    if (rc != BM25X_OK) return rc;
    BM25X_CUDA_TRY(cudaMemset((void *)(d.post + pp), 0xFF, BM25X_POST_SLACK * sizeof(Posting)));  // the slack slots read as exhausted cursors
    BM25X_CUDA_TRY(cudaMemcpy(d.post_off, h_off_pad.data(), sizeof(uint64_t) * (T + 1), cudaMemcpyHostToDevice));
    BM25X_CUDA_TRY(cudaMemcpy(d.blk_off, h_blk_off.data(), sizeof(uint64_t) * (T + 1), cudaMemcpyHostToDevice));
    if (T) {
        BM25X_CUDA_TRY(cudaMemcpy(d.df, ix->h_df.data(), sizeof(uint32_t) * T, cudaMemcpyHostToDevice));
        BM25X_CUDA_TRY(cudaMemcpy(d.s0d, st.s0d.data(), sizeof(double) * T, cudaMemcpyHostToDevice));
        BM25X_CUDA_TRY(cudaMemcpy(d.s0f, st.s0f.data(), sizeof(float) * T, cudaMemcpyHostToDevice));
    }
    BM25X_CUDA_TRY(cudaMemcpy(d.s1d, st.s1d, sizeof(st.s1d), cudaMemcpyHostToDevice));
    BM25X_CUDA_TRY(cudaMemcpy(d.s1f, st.s1f, sizeof(st.s1f), cudaMemcpyHostToDevice));
    BM25X_CUDA_TRY(cudaMemcpy(d.fieldnorm, h_fn.data(), N, cudaMemcpyHostToDevice));
    if (m.payload) {
        BM25X_CUDA_TRY(cudaMemcpy(d.payload, m.payload, sizeof(uint16_t) * 3 * (size_t)N, cudaMemcpyHostToDevice));
    } else {
        std::vector<uint16_t> pl((size_t)N * 3);
        for (uint32_t i = 0; i < N; i++) {  // synthetic ctid: (block hi, block lo, offset) of a 291-tuple page
            const uint32_t g = m.doc_base + i;  // of the segment's doc id (a shard's local ids start at doc_base)
            uint32_t blkno = g / 291;
            pl[(size_t)i * 3 + 0] = (uint16_t)(blkno >> 16);
            pl[(size_t)i * 3 + 1] = (uint16_t)(blkno & 0xFFFF);
            pl[(size_t)i * 3 + 2] = (uint16_t)(g % 291 + 1);
        }
        BM25X_CUDA_TRY(cudaMemcpy(d.payload, pl.data(), sizeof(uint16_t) * pl.size(), cudaMemcpyHostToDevice));
    }
    return BM25X_OK;
}

// After the postings are in place: pad slots, block descriptors, per-term score bounds.
static cudaError_t index_finish_device(bm25x_index *ix) {
    DeviceIndex &d = ix->d;
    const uint32_t T = d.n_terms;
    const uint64_t nb = d.n_blocks;
    cudaError_t e = cudaSuccess;
    if (T) {
        k_pad_slots<<<(T + 255) / 256, 256>>>(d.post_off, d.df, T, d.post);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        k_extract_docs<<<ix->sm_count * 8, 256>>>(d.post, d.n_post_pad + BM25X_POST_SLACK, d.pdoc);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && nb) {
        k_block_desc<<<(unsigned)((nb + 255) / 256), 256>>>(d.post_off, d.df, d.blk_off, T, nb, d.post, d.s0d, d.s1d, d.blk,
                                                            d.blk_ub);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && T) {
        k_term_ub<<<(unsigned)std::min<uint32_t>(T, (uint32_t)ix->sm_count * 16u), 256>>>(d.post_off, d.df, d.post, d.s0d, d.s1d, T, d.ubd);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = build_champions(ix);
    return e;
}

// Postings of a term-major CSR: chunked H2D of the columns + device transform to the padded AoS, then the derived arrays.
static int upload_csr(bm25x_index *ix, const char *who, uint32_t T, uint64_t P, const uint64_t *post_off,
                      const uint32_t *post_doc, const uint32_t *post_tf) {
    DeviceIndex &d = ix->d;
    const uint64_t CH = 64ull << 20;  // postings per chunk
    Scratch sc(ix->device);
    const uint64_t *d_off = sc.up(post_off, (size_t)T + 1);
    uint32_t *d_cdoc = sc.alloc<uint32_t>(std::min<uint64_t>(CH, P)), *d_ctf = sc.alloc<uint32_t>(std::min<uint64_t>(CH, P));
    for (uint64_t base = 0; base < P && sc.e == cudaSuccess; base += CH) {
        const uint64_t n = std::min<uint64_t>(CH, P - base);
        sc.e = cudaMemcpy(d_cdoc, post_doc + base, sizeof(uint32_t) * n, cudaMemcpyHostToDevice);
        if (sc.e == cudaSuccess) sc.e = cudaMemcpy(d_ctf, post_tf + base, sizeof(uint32_t) * n, cudaMemcpyHostToDevice);
        if (sc.e == cudaSuccess) {
            k_build_postings<<<(unsigned)((n + 255) / 256), 256>>>(d_cdoc, d_ctf, base, n, d_off, d.post_off, T, d.fieldnorm,
                                                                   d.post);
            sc.e = cudaGetLastError();
        }
        if (sc.e == cudaSuccess) sc.e = cudaDeviceSynchronize();
    }
    if (sc.e == cudaSuccess) sc.e = index_finish_device(ix);
    return sc.e == cudaSuccess ? BM25X_OK : cuda_refusal(who, "posting upload", sc.e);
}

// Host validation of a term-major CSR corpus, shared by bm25x_index_create and bm25x_sharded_create: same codes, same
// messages.  check_device == false leaves the device check to the caller (bm25x_sharded_create checks its shard
// arguments first, so that they are refused without a GPU).
static int validate_corpus(const bm25x_corpus *c, int device, bool check_device) {
    if (!c->post_off || (c->post_off[c->n_terms] && (!c->post_doc || !c->post_tf))) {
        bm25x_set_error("bm25x_index_create: empty or malformed corpus");
        return BM25X_ERR_INVALID;
    }
    int rc = check_common("bm25x_index_create", c->n_docs, c->doc_len, c->k1, c->b, device);
    if (rc != BM25X_OK && (check_device || rc != BM25X_ERR_CUDA)) return rc;
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t P = c->post_off[T];

    // ---- host-side validation of the CSR (the reference panics with "data corruption") ----
    int bad = 0;  // 1 = ordering/ranges, 2 = tf too large
#pragma omp parallel for schedule(dynamic, 256) reduction(| : bad) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++) {
        uint64_t p0 = c->post_off[t], p1 = c->post_off[t + 1];
        if (p1 < p0 || p1 > P) {
            bad |= 1;
            continue;
        }
        if (p1 - p0 > N) bad |= 1;
        uint32_t prev = 0;
        for (uint64_t p = p0; p < p1; p++) {
            uint32_t d = c->post_doc[p], f = c->post_tf[p];
            if (d >= N || f == 0 || (p > p0 && d <= prev)) bad |= 1;
            if (f >= (1u << 24)) bad |= 2;
            prev = d;
        }
    }
    if (bad & 1) {
        bm25x_set_error("bm25x_index_create: corrupt corpus (doc ids must be < n_docs and strictly ascending per term, tf != 0)");
        return BM25X_ERR_INVALID;
    }
    if (bad & 2) {
        bm25x_set_error("bm25x_index_create: term frequency >= 2^24 is not supported by the packed posting layout");
        return BM25X_ERR_UNSUPPORTED;
    }
    return check_keys("bm25x_index_create", c->term_key, T);
}

extern "C" int bm25x_index_create(const bm25x_corpus *c, int device, bm25x_index **out) {
    if (!c || !out) {
        bm25x_set_error("bm25x_index_create: null argument");
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    int rc = validate_corpus(c, device, true);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t P = c->post_off[T];

    std::vector<uint32_t> df(T);
    for (uint32_t t = 0; t < T; t++) df[t] = (uint32_t)(c->post_off[t + 1] - c->post_off[t]);
    BuildMeta m{N, T, c->doc_len, c->payload, c->term_key, c->k1, c->b, df.data(), P};
    IndexGuard ix;
    rc = index_begin(m, nullptr, device, ix);
    if (rc == BM25X_OK) rc = upload_csr(ix.get(), "bm25x_index_create", T, P, c->post_off, c->post_doc, c->post_tf);
    if (rc == BM25X_OK) *out = ix.release();
    return rc;
}

// ---- document-sharded index (DESIGN §4.7): one segment split by document range, each shard an index with local doc ids
// that scores with the whole segment's statistics ----
extern "C" void bm25x_sharded_destroy(bm25x_sharded_index *sx) {
    if (!sx) return;
    for (bm25x_index *ix : sx->shards) bm25x_index_destroy(ix);
    delete sx;
}

// The shard arguments of a document-sharded build, by bm25x_sharded_create's rules and with its messages whichever entry
// point is called: 1..BM25X_MAX_SHARDS shards, at least one document each, explicit bounds strictly ascending from 0 to N.
static int check_shard_args(uint32_t N, uint32_t S, const uint32_t *doc_bounds) {
    const char *who = "bm25x_sharded_create";
    if (S == 0 || S > BM25X_MAX_SHARDS) {
        bm25x_set_error("%s: n_shards=%u must be 1..%d", who, S, BM25X_MAX_SHARDS);
        return BM25X_ERR_INVALID;
    }
    if (N < S) {
        bm25x_set_error("%s: n_docs=%u < n_shards=%u (every shard holds at least one document)", who, N, S);
        return BM25X_ERR_INVALID;
    }
    if (doc_bounds) {
        bool ok = doc_bounds[0] == 0 && doc_bounds[S] == N;
        for (uint32_t s = 0; s < S && ok; s++) ok = doc_bounds[s] < doc_bounds[s + 1];
        if (!ok) {
            bm25x_set_error("%s: doc_bounds must ascend strictly from 0 to n_docs=%u", who, N);
            return BM25X_ERR_INVALID;
        }
    }
    return BM25X_OK;
}

// The shard bounds of a document-sharded build: doc_bounds as given (checked by check_shard_args), or, when it is NULL,
// balanced by postings from cum[d] = Σ_{d' < d} c_{d'} (c_d = distinct terms of document d = its postings; cum[N] = P):
// b_s = smallest d > b_{s-1} with cum[d] >= ceil(s·P/S), clamped so that the shards s..S-1 keep one document each.
static std::vector<uint32_t> shard_bounds(const uint32_t *doc_bounds, const std::vector<uint64_t> &cum, uint32_t N,
                                          uint32_t S) {
    std::vector<uint32_t> bounds((size_t)S + 1);
    if (doc_bounds) {
        std::copy(doc_bounds, doc_bounds + S + 1, bounds.begin());
        return bounds;
    }
    const uint64_t P = cum[N];
    bounds[0] = 0;
    for (uint32_t s = 1; s < S; s++) {
        const uint64_t target = ((uint64_t)s * P + S - 1) / S;
        // smallest d > b_{s-1} with cum[d] >= target (cum ascends; cum[N] = P >= target)
        uint32_t d = (uint32_t)(std::lower_bound(cum.begin() + bounds[s - 1] + 1, cum.end(), target) - cum.begin());
        bounds[s] = std::min<uint32_t>(d, N - (S - s));
    }
    bounds[S] = N;
    return bounds;
}

// The container of a document-sharded build, for both sources: after the host checks of the segment c (P postings, df, the
// statistics st), every shard's device is checked with who's message; then prepare(device of shard 0, cum) runs the
// host work and refusals that need a device and, when doc_bounds is NULL, gives the postings per document for the balanced
// bounds (shard_bounds); then the shards are built one at a time by build(s, device, lo, hi, ix).  On the first failure
// everything built so far is destroyed.
template <typename Segment, typename Prepare, typename Build>
static int sharded_build(const char *who, const Segment *c, uint64_t P, const std::vector<uint32_t> &df, const Stats &st,
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

extern "C" int bm25x_sharded_create(const bm25x_corpus *c, uint32_t S, const uint32_t *doc_bounds, const int *devices,
                                    bm25x_sharded_index **out) {
    const char *who = "bm25x_sharded_create";
    if (!c || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    // every host check before any device is used: the corpus exactly as bm25x_index_create checks it, then the shards
    int rc = validate_corpus(c, 0, false);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t P = c->post_off[T];
    rc = check_shard_args(N, S, doc_bounds);
    if (rc != BM25X_OK) return rc;
    std::vector<uint32_t> df(T);
    for (uint32_t t = 0; t < T; t++) df[t] = (uint32_t)(c->post_off[t + 1] - c->post_off[t]);
    const Stats st(N, doc_norms(N, c->doc_len, nullptr, 0, nullptr), df.data(), T, c->k1, c->b);
    auto count = [&](int, std::vector<uint64_t> *cum) {
        if (!cum) return BM25X_OK;
        cum->assign((size_t)N + 1, 0);
#pragma omp parallel for schedule(static) num_threads(bm25x_host_threads(0))
        for (uint64_t p = 0; p < P; p++) {
#pragma omp atomic
            (*cum)[(size_t)c->post_doc[p] + 1]++;
        }
        for (uint32_t d = 0; d < N; d++) (*cum)[(size_t)d + 1] += (*cum)[d];
        return BM25X_OK;
    };
    // one shard at a time: host memory beyond the corpus stays within one shard's CSR
    auto build = [&](uint32_t s, int device, uint32_t lo, uint32_t hi, IndexGuard &ix) {
        std::vector<uint64_t> off((size_t)T + 1, 0);
        std::vector<uint64_t> first(T);
#pragma omp parallel for schedule(dynamic, 256) num_threads(bm25x_host_threads(0))
        for (uint32_t t = 0; t < T; t++) {  // the shard's range inside the term's (ascending) list
            const uint32_t *a = c->post_doc + c->post_off[t], *e = c->post_doc + c->post_off[t + 1];
            const uint32_t *p0 = std::lower_bound(a, e, lo), *p1 = std::lower_bound(p0, e, hi);
            first[t] = (uint64_t)(p0 - c->post_doc);
            off[(size_t)t + 1] = (uint64_t)(p1 - p0);
        }
        std::vector<uint32_t> df_s(T);
        for (uint32_t t = 0; t < T; t++) {
            df_s[t] = (uint32_t)off[(size_t)t + 1];
            off[(size_t)t + 1] += off[t];
        }
        const uint64_t Ps = off[T];
        std::vector<uint32_t> pdoc(Ps ? Ps : 1), ptf(Ps ? Ps : 1);
#pragma omp parallel for schedule(dynamic, 256) num_threads(bm25x_host_threads(0))
        for (uint32_t t = 0; t < T; t++)
            for (uint64_t i = 0; i < off[(size_t)t + 1] - off[t]; i++) {
                pdoc[off[t] + i] = c->post_doc[first[t] + i] - lo;
                ptf[off[t] + i] = c->post_tf[first[t] + i];
            }
        // (the term keys once, with shard 0: bm25x_sharded_lookup_terms asks it)
        BuildMeta m{hi - lo, T, c->doc_len + lo, c->payload ? c->payload + (size_t)lo * 3 : nullptr, s ? nullptr : c->term_key,
                    c->k1, c->b, df_s.data(), Ps};
        m.doc_base = lo;
        const int rc = index_begin(m, &st, device, ix);
        return rc == BM25X_OK ? upload_csr(ix.get(), who, T, Ps, off.data(), pdoc.data(), ptf.data()) : rc;
    };
    return sharded_build(who, c, P, df, st, S, doc_bounds, devices, count, build, out);
}

// ---- f1: the sealed segment as the reference stores it (blocks in the codec of compression.rs), decoded on the GPU ----

// Host validation of the stored blocks, shared by bm25x_index_create_from_blocks and
// bm25x_index_create_sharded_from_blocks: same codes, same messages.  Gives each token's postings (df) and their total P.
// check_device == false leaves the device check to the caller (the sharded build checks its shard arguments first, so
// that they are refused without a GPU).
static int validate_blocks(const bm25x_blocks *c, int device, bool check_device, std::vector<uint32_t> &df,
                           uint64_t &n_post) {
    const char *who = "bm25x_index_create_from_blocks";
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t NB = c->n_blocks;
    if (!c->term_blk_off || (NB && (!c->blk_min_doc || !c->blk_n || !c->blk_meta_doc || !c->blk_meta_tf ||
                                    !c->blk_doc_off || !c->blk_tf_off || (c->n_bytes && !c->bytes)))) {
        bm25x_set_error("%s: empty or malformed corpus", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_common(who, N, c->doc_len ? (const void *)c->doc_len : (const void *)c->doc_fieldnorm, c->k1, c->b, device);
    if (rc != BM25X_OK && (check_device || rc != BM25X_ERR_CUDA)) return rc;
    if (c->term_blk_off[0] != 0 || c->term_blk_off[T] != NB) {
        bm25x_set_error("%s: term_blk_off must run from 0 to n_blocks", who);
        return BM25X_ERR_INVALID;
    }
    // ---- host-side validation of the block directory (payloads are validated by the decoder on the device) ----
    df.assign(T, 0);
    uint64_t P = 0;
    int bad = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(| : bad) reduction(+ : P) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++) {
        const uint64_t b0 = c->term_blk_off[t], b1 = c->term_blk_off[t + 1];
        if (b1 < b0 || b1 > NB) {
            bad |= 1;
            df[t] = 0;
            continue;
        }
        uint64_t n_t = 0;
        for (uint64_t g = b0; g < b1; g++) {
            const uint32_t n = c->blk_n[g];
            // flush.rs:80-90: every block of a token holds 128 postings except the last one
            if (n == 0 || n > BM25X_BLOCK || (n < BM25X_BLOCK && g + 1 != b1)) bad |= 1;
            const uint8_t metas[2] = {c->blk_meta_doc[g], c->blk_meta_tf[g]};
            const uint64_t offs[2] = {c->blk_doc_off[g], c->blk_tf_off[g]};
            for (int s = 0; s < 2; s++) {
                const uint32_t w = metas[s] & 0x7Fu;
                uint64_t nbytes;
                if ((metas[s] >> 7) == 0) {  // compression.rs:43-52: bit packing only for full blocks, width <= 32
                    if (w > 32 || n != BM25X_BLOCK) bad |= 2;
                    nbytes = (uint64_t)w * 16;
                } else {                      // compression.rs:53-62: 1..4 bytes per value
                    if (w < 1 || w > 4) bad |= 2;
                    nbytes = (uint64_t)w * n;
                }
                if (offs[s] > c->n_bytes || nbytes > c->n_bytes - offs[s]) bad |= 1;
            }
            n_t += n;
        }
        if (n_t > N) bad |= 1;
        df[t] = (uint32_t)std::min<uint64_t>(n_t, N);
        P += n_t;
    }
    if (bad & 1) {
        bm25x_set_error("%s: corrupt block directory (block sizes, token ranges or payload offsets)", who);
        return BM25X_ERR_INVALID;
    }
    if (bad & 2) {
        bm25x_set_error("%s: corrupt block metadata (bitwidth out of bound / unexpected input len)", who);
        return BM25X_ERR_INVALID;
    }
    n_post = P;
    return check_keys(who, c->term_key, T);
}

// The refusal for the error bits of the decode and check kernels (bm25x_blocks.cuh), with the messages of
// bm25x_index_create_from_blocks whichever entry point decoded the blocks.
static int blocks_refusal(uint32_t h_err) {
    const char *who = "bm25x_index_create_from_blocks";
    if (h_err & BM25X_BLKERR_RANGE) {
        bm25x_set_error("%s: corrupt blocks (doc ids must be < n_docs and strictly ascending per token, tf != 0)", who);
        return BM25X_ERR_INVALID;
    }
    if (h_err & BM25X_BLKERR_TF) {
        bm25x_set_error("%s: term frequency >= 2^24 is not supported by the packed posting layout", who);
        return BM25X_ERR_UNSUPPORTED;
    }
    if (h_err & BM25X_BLKERR_WAND) {
        bm25x_set_error("%s: corrupt blocks (SummaryTuple wand_fieldnorm/wand_term_frequency is not the block's maximum)", who);
        return BM25X_ERR_INVALID;
    }
    if (h_err & BM25X_BLKERR_DIR) {  // only blocks staged by the sharded build: the caller's directory changed under it
        bm25x_set_error("%s: corrupt block directory (block sizes, token ranges or payload offsets)", who);
        return BM25X_ERR_INVALID;
    }
    return BM25X_OK;
}

extern "C" int bm25x_index_create_from_blocks(const bm25x_blocks *c, int device, bm25x_index **out) {
    const char *who = "bm25x_index_create_from_blocks";
    if (!c || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    std::vector<uint32_t> df;
    uint64_t P = 0;
    int rc = validate_blocks(c, device, true, df, P);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t NB = c->n_blocks;

    BuildMeta m{N, T, c->doc_len, c->payload, c->term_key, c->k1, c->b, df.data(), P};
    m.fieldnorm = c->doc_fieldnorm;
    m.sum_len = c->sum_doc_len;
    IndexGuard ix;
    rc = index_begin(m, nullptr, device, ix);
    if (rc != BM25X_OK) return rc;
    DeviceIndex &d = ix->d;

    // ---- upload the directory + payloads, decode on the device ----
    uint32_t h_err = 0;
    Scratch sc(device);
    const uint64_t *d_tbo = sc.up(c->term_blk_off, (size_t)T + 1);
    const uint32_t *d_min = sc.up(c->blk_min_doc, NB), *d_n = sc.up(c->blk_n, NB);
    const uint8_t *d_md = sc.up(c->blk_meta_doc, NB), *d_mt = sc.up(c->blk_meta_tf, NB);
    const uint64_t *d_doff = sc.up(c->blk_doc_off, NB), *d_toff = sc.up(c->blk_tf_off, NB);
    const uint8_t *d_bytes = sc.up(c->bytes, c->n_bytes);
    uint32_t *d_err = sc.up(&h_err, 1);
    if (sc.e == cudaSuccess && NB) {
        k_decode_blocks<<<(unsigned)((NB + DEC_WARPS - 1) / DEC_WARPS), DEC_WARPS * 32>>>(
            NB, d_tbo, T, d_min, d_n, d_md, d_mt, d_doff, d_toff, d_bytes, d.post_off, d.fieldnorm, N, d.post, d_err);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = index_finish_device(ix.get());
    if (c->blk_wand_fieldnorm && c->blk_wand_tf) {  // the stored per-block bounds must be those of the decoded postings
        const uint8_t *d_wfn = sc.up(c->blk_wand_fieldnorm, NB);
        const uint32_t *d_wtf = sc.up(c->blk_wand_tf, NB);
        if (sc.e == cudaSuccess && NB) {
            k_check_block_wand<<<(unsigned)((NB + 255) / 256), 256>>>(NB, d.blk_off, T, d_wfn, d_wtf, d.s0d, d.s1d, d.blk_ub,
                                                                     d_err);
            sc.e = cudaGetLastError();
        }
    }
    if (sc.e == cudaSuccess && NB > 1) {
        k_check_block_order<<<(unsigned)((NB + 255) / 256), 256>>>(d.blk_off, T, NB, d.blk, d_err);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "block upload/decode", sc.e);
    rc = blocks_refusal(h_err);
    if (rc == BM25X_OK) *out = ix.release();
    return rc;
}

// ---- a document-sharded index from the stored blocks (DESIGN §4.7): one check pass over the whole segment on shard 0's
// device, then per shard a decode of just the stored blocks that hold its documents, on its own device ----

// Directory entries and payloads of some stored blocks, gathered back to back with the offsets rebased to `bytes`: what a
// kernel of bm25x_blocks.cuh reads for just these blocks.  The directory has passed validate_blocks.
struct StagedBlocks {
    std::vector<uint32_t> min, n;
    std::vector<uint8_t> md, mt;
    std::vector<uint64_t> doff, toff;
    std::vector<uint8_t> bytes;

    void gather(const bm25x_blocks *c, const uint64_t *ids, size_t nb) {
        min.resize(nb);
        n.resize(nb);
        md.resize(nb);
        mt.resize(nb);
        doff.resize(nb);
        toff.resize(nb);
        uint64_t pos = 0;
        for (size_t j = 0; j < nb; j++) {
            const uint64_t g = ids[j];
            min[j] = c->blk_min_doc[g];
            n[j] = c->blk_n[g];
            md[j] = c->blk_meta_doc[g];
            mt[j] = c->blk_meta_tf[g];
            doff[j] = pos;
            pos += stream_bytes(md[j], n[j]);
            toff[j] = pos;
            pos += stream_bytes(mt[j], n[j]);
        }
        bytes.resize(pos ? pos : 1);
        n_bytes = pos;
#pragma omp parallel for schedule(static) num_threads(bm25x_host_threads(0))
        for (size_t j = 0; j < nb; j++) {
            const uint64_t g = ids[j];
            memcpy(bytes.data() + doff[j], c->bytes + c->blk_doc_off[g], toff[j] - doff[j]);
            memcpy(bytes.data() + toff[j], c->bytes + c->blk_tf_off[g], stream_bytes(mt[j], n[j]));
        }
    }
    uint64_t n_bytes = 0;
};

// The check pass: every stored block decoded once on `device`, in chunks of at most 256 MiB of payload (so the compressed
// segment never has to fit on one GPU), with every check bm25x_index_create_from_blocks makes on the device.  Gives the
// error bits, each block's decoded (first, last) doc id, and with cum != NULL the postings of the documents < d (cum[d]).
// fieldnorm and the s0 / s1 tables of stats are the segment's; they are read only to check the stored wand pairs.
static int check_stored_blocks(const char *who, const bm25x_blocks *c, const uint8_t *fieldnorm, const Stats &stats,
                               int device, std::vector<uint2> &first_last, std::vector<uint64_t> *cum, uint32_t &h_err) {
    const uint32_t N = c->n_docs, T = c->n_terms;
    const uint64_t NB = c->n_blocks;
    const bool wand = c->blk_wand_fieldnorm && c->blk_wand_tf;
    first_last.assign(NB, make_uint2(0, 0));
    h_err = 0;
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const uint64_t *d_tbo = sc.up(c->term_blk_off, (size_t)T + 1);
    const uint8_t *d_fn = wand ? sc.up(fieldnorm, N) : nullptr;  // the whole segment's norms: a block may straddle a bound
    const double *d_s0d = wand ? sc.up(stats.s0d.data(), T) : nullptr;
    const double *d_s1d = wand ? sc.up(stats.s1d, 256) : nullptr;
    uint32_t *d_cnt = cum ? sc.alloc<uint32_t>(N) : nullptr;
    if (d_cnt && sc.e == cudaSuccess) sc.e = cudaMemset(d_cnt, 0, sizeof(uint32_t) * (size_t)N);
    uint32_t *d_err = sc.up(&h_err, 1);
    const uint64_t CH_BYTES = 256ull << 20, CH_BLOCKS = 1ull << 21;
    std::vector<uint64_t> ids;
    StagedBlocks st;
    for (uint64_t g0 = 0; g0 < NB && sc.e == cudaSuccess;) {
        uint64_t g1 = g0, nbytes = 0;
        while (g1 < NB && g1 - g0 < CH_BLOCKS) {
            const uint64_t b = (uint64_t)stream_bytes(c->blk_meta_doc[g1], c->blk_n[g1]) +
                               stream_bytes(c->blk_meta_tf[g1], c->blk_n[g1]);
            if (g1 > g0 && nbytes + b > CH_BYTES) break;
            nbytes += b;
            g1++;
        }
        const uint64_t nb = g1 - g0;
        ids.resize(nb);
        for (uint64_t j = 0; j < nb; j++) ids[j] = g0 + j;
        st.gather(c, ids.data(), nb);
        Scratch ch(device);
        const uint32_t *d_min = ch.up(st.min.data(), nb), *d_n = ch.up(st.n.data(), nb);
        const uint8_t *d_md = ch.up(st.md.data(), nb), *d_mt = ch.up(st.mt.data(), nb);
        const uint64_t *d_doff = ch.up(st.doff.data(), nb), *d_toff = ch.up(st.toff.data(), nb);
        const uint8_t *d_bytes = ch.up(st.bytes.data(), st.bytes.size());
        const uint8_t *d_wfn = wand ? ch.up(c->blk_wand_fieldnorm + g0, nb) : nullptr;
        const uint32_t *d_wtf = wand ? ch.up(c->blk_wand_tf + g0, nb) : nullptr;
        uint2 *d_fl = ch.alloc<uint2>(nb);
        if (ch.e == cudaSuccess) {
            k_check_blocks<<<(unsigned)((nb + DEC_WARPS - 1) / DEC_WARPS), DEC_WARPS * 32>>>(
                g0, nb, d_tbo, T, d_min, d_n, d_md, d_mt, d_doff, d_toff, d_bytes, st.n_bytes, d_fn, N, d_wfn, d_wtf, d_s0d,
                d_s1d, d_fl, d_cnt, d_err);
            ch.e = cudaGetLastError();
        }
        if (ch.e == cudaSuccess) ch.e = cudaMemcpy(first_last.data() + g0, d_fl, sizeof(uint2) * nb, cudaMemcpyDeviceToHost);
        sc.e = ch.e;
        g0 = g1;
    }
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost);
    if (sc.e == cudaSuccess && cum) {
        std::vector<uint32_t> cnt(N);
        sc.e = cudaMemcpy(cnt.data(), d_cnt, sizeof(uint32_t) * (size_t)N, cudaMemcpyDeviceToHost);
        cum->assign((size_t)N + 1, 0);
        for (uint32_t d = 0; d < N; d++) (*cum)[(size_t)d + 1] = (*cum)[d] + cnt[d];
    }
    if (sc.e != cudaSuccess) return cuda_refusal(who, "block upload/decode", sc.e);
    // k_check_block_order's rule on the decoded (first, last): ids ascend across the blocks of a token
    uint32_t order = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(| : order) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++)
        for (uint64_t g = c->term_blk_off[t] + 1; g < c->term_blk_off[t + 1]; g++)
            if (first_last[g].x <= first_last[g - 1].y) order |= BM25X_BLKERR_RANGE;
    h_err |= order;
    return BM25X_OK;
}

// Shard s, documents [lo, hi), from the stored blocks, on `device`: the blocks whose decoded [first, last] meets [lo, hi)
// gathered with rebased offsets (host memory beyond the caller's: this payload), counted (k_count_shard_blocks), then the
// shard index allocated with the whole segment's statistics, decoded into place (k_decode_shard_blocks) and finished as
// every index is.
static int build_shard_from_blocks(const char *who, const bm25x_blocks *c, const std::vector<uint2> &first_last,
                                   const Stats &stats, uint32_t s, uint32_t lo, uint32_t hi, int device, IndexGuard &ix) {
    const uint32_t T = c->n_terms;
    // ---- select: per token the run of its blocks with last >= lo and first < hi (both ascend along the chain) ----
    std::vector<uint64_t> sel_b0(T), sel_off((size_t)T + 1, 0);
#pragma omp parallel for schedule(dynamic, 256) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++) {
        const uint2 *a = first_last.data() + c->term_blk_off[t], *e = first_last.data() + c->term_blk_off[t + 1];
        const uint2 *b0 = std::partition_point(a, e, [&](const uint2 &f) { return f.y < lo; });
        const uint2 *b1 = std::partition_point(b0, e, [&](const uint2 &f) { return f.x < hi; });
        sel_b0[t] = (uint64_t)(b0 - first_last.data());
        sel_off[(size_t)t + 1] = (uint64_t)(b1 - b0);
    }
    for (uint32_t t = 0; t < T; t++) sel_off[(size_t)t + 1] += sel_off[t];
    const uint64_t nsel = sel_off[T];
    std::vector<uint64_t> ids(nsel);
    std::vector<uint2> sel_fl(nsel);
#pragma omp parallel for schedule(dynamic, 256) num_threads(bm25x_host_threads(0))
    for (uint32_t t = 0; t < T; t++)
        for (uint64_t j = sel_off[t]; j < sel_off[(size_t)t + 1]; j++) {
            ids[j] = sel_b0[t] + (j - sel_off[t]);
            sel_fl[j] = first_last[ids[j]];
        }
    StagedBlocks st;
    st.gather(c, ids.data(), nsel);
    std::vector<uint64_t>().swap(ids);
    // ---- count: the shard's df, and each selected block's rank inside its token's shard list ----
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const uint32_t *d_min = sc.up(st.min.data(), nsel), *d_n = sc.up(st.n.data(), nsel);
    const uint8_t *d_md = sc.up(st.md.data(), nsel), *d_mt = sc.up(st.mt.data(), nsel);
    const uint64_t *d_doff = sc.up(st.doff.data(), nsel), *d_toff = sc.up(st.toff.data(), nsel);
    const uint8_t *d_bytes = sc.up(st.bytes.data(), st.bytes.size());
    const uint2 *d_fl = sc.up(sel_fl.data(), nsel);
    const uint64_t *d_sel_off = sc.up(sel_off.data(), (size_t)T + 1);
    uint2 *d_cs = sc.alloc<uint2>(nsel);
    uint32_t h_err = 0, *d_err = sc.up(&h_err, 1);
    const unsigned grid = (unsigned)((nsel + DEC_WARPS - 1) / DEC_WARPS);
    if (sc.e == cudaSuccess && nsel) {
        k_count_shard_blocks<<<grid, DEC_WARPS * 32>>>(nsel, d_fl, d_min, d_n, d_md, d_doff, d_bytes, st.n_bytes, lo, hi,
                                                        d_cs, d_err);
        sc.e = cudaGetLastError();
    }
    std::vector<uint2> cs(nsel);
    if (sc.e == cudaSuccess && nsel) sc.e = cudaMemcpy(cs.data(), d_cs, sizeof(uint2) * nsel, cudaMemcpyDeviceToHost);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "block upload/decode", sc.e);
    std::vector<uint32_t> df(T), rank(nsel);
    uint64_t Ps = 0;
    for (uint32_t t = 0; t < T; t++) {
        uint64_t run = 0;
        for (uint64_t j = sel_off[t]; j < sel_off[(size_t)t + 1]; j++) {
            rank[j] = (uint32_t)std::min<uint64_t>(run, 0xFFFFFFFFu);
            run += cs[j].x;
        }
        df[t] = (uint32_t)std::min<uint64_t>(run, hi - lo);  // more than the shard's documents: refused by the decode
        Ps += df[t];
    }
    // ---- allocate the shard as bm25x_sharded_create does (the term keys once, with shard 0) ----
    BuildMeta m{hi - lo, T, c->doc_len ? c->doc_len + lo : nullptr, c->payload ? c->payload + (size_t)lo * 3 : nullptr,
                s ? nullptr : c->term_key, c->k1, c->b, df.data(), Ps};
    m.fieldnorm = c->doc_len ? nullptr : c->doc_fieldnorm + lo;
    m.sum_len = c->sum_doc_len;  // stored norms: the pages hold the segment's sum only
    m.doc_base = lo;
    const int rc = index_begin(m, &stats, device, ix);
    if (rc != BM25X_OK) return rc;
    // ---- write the postings, then what every index derives from them ----
    const uint32_t *d_rank = sc.up(rank.data(), nsel);
    if (sc.e == cudaSuccess && nsel) {
        k_decode_shard_blocks<<<grid, DEC_WARPS * 32>>>(nsel, d_sel_off, T, d_min, d_n, d_md, d_mt, d_doff, d_toff, d_bytes,
                                                         st.n_bytes, d_cs, d_rank, c->n_docs, lo, hi - lo,
                                                         ix->d.post_off, ix->d.df, ix->d.fieldnorm, ix->d.post, d_err);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&h_err, d_err, sizeof(h_err), cudaMemcpyDeviceToHost);
    if (sc.e == cudaSuccess && !h_err) sc.e = index_finish_device(ix.get());
    return sc.e != cudaSuccess ? cuda_refusal(who, "block upload/decode", sc.e) : blocks_refusal(h_err);
}

extern "C" int bm25x_index_create_sharded_from_blocks(const bm25x_blocks *c, uint32_t S, const uint32_t *doc_bounds,
                                                      const int *devices, bm25x_sharded_index **out) {
    const char *who = "bm25x_index_create_sharded_from_blocks";
    if (!c || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    // every host check before any device is used: the blocks exactly as bm25x_index_create_from_blocks checks them, then
    // the shard arguments exactly as bm25x_sharded_create checks them
    std::vector<uint32_t> df;
    uint64_t P = 0;
    int rc = validate_blocks(c, 0, false, df, P);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = c->n_docs, T = c->n_terms;
    rc = check_shard_args(N, S, doc_bounds);
    if (rc != BM25X_OK) return rc;
    // the segment's norms (the stored ones, or quantised for the check pass) and statistics
    std::vector<uint8_t> h_fn(c->doc_len ? N : 0);
    const uint8_t *fn = c->doc_len ? h_fn.data() : c->doc_fieldnorm;
    const Stats st(N, doc_norms(N, c->doc_len, c->doc_fieldnorm, c->sum_doc_len, c->doc_len ? h_fn.data() : nullptr),
                   df.data(), T, c->k1, c->b);
    std::vector<uint2> first_last;
    // ---- check pass on shard 0's device: the refusals of the unsharded ingest, before any shard exists ----
    auto check = [&](int device, std::vector<uint64_t> *cum) {
        uint32_t h_err = 0;
        const int rc = check_stored_blocks(who, c, fn, st, device, first_last, cum, h_err);
        std::vector<uint8_t>().swap(h_fn);
        return rc != BM25X_OK ? rc : blocks_refusal(h_err);
    };
    // one shard at a time: host memory beyond the blocks stays within one shard's selected payload
    auto build = [&](uint32_t s, int device, uint32_t lo, uint32_t hi, IndexGuard &ix) {
        return build_shard_from_blocks(who, c, first_last, st, s, lo, hi, device, ix);
    };
    return sharded_build(who, c, P, df, st, S, doc_bounds, devices, check, build, out);
}

// ---- f3: the growing segment (documents inserted since the last seal, search.rs:83-135) as a second, small index that
// scores with the sealed segment's statistics.  The reference scans these documents one by one per query; here they
// are inverted once (term-major postings over growing ordinals) so that the same kernels unite them. ----
extern "C" int bm25x_growing_create(const bm25x_index *sealed, const bm25x_growing_docs *g, bm25x_index **out) {
    const char *who = "bm25x_growing_create";
    if (!sealed || !g || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    const uint32_t G = g->n_docs, T = sealed->d.n_terms;
    if (!g->elem_off || (g->elem_off[G] && (!g->elem_term || !g->elem_tf))) {
        bm25x_set_error("%s: empty or malformed corpus", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_common(who, G, g->doc_len ? (const void *)g->doc_len : (const void *)g->doc_fieldnorm, sealed->k1,
                          sealed->b, sealed->device);
    if (rc != BM25X_OK) return rc;
    // growing documents come back as sealed n_docs + ordinal (bm25x_search_batch_growing): the sum obeys check_common's
    // bound on n_docs, so that every merged id stays below the BM25X_DOC_INF sentinel
    if ((uint64_t)sealed->d.n_docs + G > (uint64_t)BM25X_DOC_INF - 1u) {
        bm25x_set_error("%s: sealed n_docs=%u + growing n_docs=%u exceeds %u documents (doc ids are 32-bit, %u is reserved)",
                        who, sealed->d.n_docs, G, BM25X_DOC_INF - 1u, BM25X_DOC_INF);
        return BM25X_ERR_INVALID;
    }
    // pass 1: validate the documents (vector.rs:39-75: keys strictly ascending, tf != 0) and count per-term postings
    std::vector<uint64_t> off((size_t)T + 1, 0);
    int bad = 0;
    for (uint32_t d = 0; d < G; d++) {
        const uint64_t e0 = g->elem_off[d], e1 = g->elem_off[d + 1];
        if (e1 < e0 || e1 > g->elem_off[G]) {
            bad |= 1;
            break;
        }
        if (g->deleted && g->deleted[d]) continue;  // VectorTuple.deleted (search.rs:110)
        bool have_prev = false;
        uint32_t prev = 0;
        for (uint64_t e = e0; e < e1; e++) {
            const uint32_t t = g->elem_term[e], f = g->elem_tf[e];
            if (f == 0) bad |= 1;
            if (t == BM25X_TERM_MISSING) continue;  // token unknown to the sealed segment: never matches (search.rs:60-62)
            if (have_prev && t <= prev) bad |= 1;
            have_prev = true;
            prev = t;
            if (t >= T || sealed->h_df[t] == 0) continue;
            if (f >= (1u << 24)) bad |= 2;
            off[(size_t)t + 1]++;
        }
    }
    if (bad & 1) {
        bm25x_set_error("%s: corrupt documents (term ordinals must be strictly ascending per document, tf != 0)", who);
        return BM25X_ERR_INVALID;
    }
    if (bad & 2) {
        bm25x_set_error("%s: term frequency >= 2^24 is not supported by the packed posting layout", who);
        return BM25X_ERR_UNSUPPORTED;
    }
    std::vector<uint32_t> df(T);
    for (uint32_t t = 0; t < T; t++) {
        df[t] = (uint32_t)off[(size_t)t + 1];
        off[(size_t)t + 1] += off[t];
    }
    const uint64_t P = off[T];
    // pass 2: invert (documents are visited in ascending ordinal, so every term's list comes out ascending)
    std::vector<uint32_t> post_doc(P ? P : 1), post_tf(P ? P : 1);
    {
        std::vector<uint64_t> cur(off.begin(), off.end() - 1);
        for (uint32_t d = 0; d < G; d++) {
            if (g->deleted && g->deleted[d]) continue;
            for (uint64_t e = g->elem_off[d]; e < g->elem_off[d + 1]; e++) {
                const uint32_t t = g->elem_term[e];
                if (t == BM25X_TERM_MISSING || t >= T || sealed->h_df[t] == 0) continue;
                post_doc[cur[t]] = d;
                post_tf[cur[t]] = g->elem_tf[e];
                cur[t]++;
            }
        }
    }
    BuildMeta m{G, T, g->doc_len, g->payload, sealed->h_keys.empty() ? nullptr : sealed->h_keys.data(), sealed->k1,
                sealed->b, df.data(), P};
    m.fieldnorm = g->doc_fieldnorm;
    // search.rs:66-77: scored with the SEALED segment's statistics, not its own
    const Stats st(sealed->d.n_docs, sealed->sum_len, sealed->avgdl, sealed->h_df.data(), T, sealed->k1, sealed->b);
    IndexGuard ix;
    rc = index_begin(m, &st, sealed->device, ix);
    if (rc == BM25X_OK) rc = upload_csr(ix.get(), who, T, P, off.data(), post_doc.data(), post_tf.data());
    if (rc != BM25X_OK) return rc;
    ix->prune = sealed->prune;
    *out = ix.release();
    return BM25X_OK;
}

extern "C" void bm25x_index_destroy(bm25x_index *ix) {
    if (!ix) return;
    cudaSetDevice(ix->device);
    if (ix->stream) cudaStreamSynchronize(ix->stream);
    for (void *p : ix->allocs) cudaFree(p);
    if (ix->h_stage) cudaFreeHost(ix->h_stage);
    if (ix->h_stage_free) cudaEventDestroy(ix->h_stage_free);
    if (ix->copy_stream) cudaStreamDestroy(ix->copy_stream);
    if (ix->stream) cudaStreamDestroy(ix->stream);
    delete ix;
}

extern "C" int bm25x_index_get_info(const bm25x_index *ix, bm25x_index_info *out) {
    if (!ix || !out) {
        bm25x_set_error("bm25x_index_get_info: null argument");
        return BM25X_ERR_INVALID;
    }
    out->n_docs = ix->d.n_docs;
    out->n_terms = ix->d.n_terms;
    out->n_postings = ix->d.n_post;
    out->sum_doc_len = ix->sum_len;
    out->avgdl = ix->avgdl;
    out->k1 = ix->k1;
    out->b = ix->b;
    out->device_bytes = ix->device_bytes;
    out->n_blocks = ix->d.n_blocks;
    out->device = ix->device;
    return BM25X_OK;
}

// ---- replication: expose / adopt the device arrays (the bytes travel by NCCL in the caller) ----
static void layout_arrays(const bm25x_index *ix, void **ptr, uint64_t *bytes) {
    const DeviceIndex &d = ix->d;
    const uint64_t T = d.n_terms, N = d.n_docs;
    void *p[BM25X_N_ARRAYS] = {d.post, d.post_off, d.df, d.blk_off, d.blk, d.s0f, d.s0d, d.s1d, d.s1f, d.fieldnorm, d.payload,
                               d.ubd, d.blk_ub};
    uint64_t b[BM25X_N_ARRAYS] = {sizeof(Posting) * (d.n_post_pad + BM25X_POST_SLACK), 8 * (T + 1), 4 * (T ? T : 1), 8 * (T + 1),
                                  8 * (d.n_blocks ? d.n_blocks : 1), 4 * (T ? T : 1), 8 * (T ? T : 1), 8 * 256, 4 * 256,
                                  N, 6 * N, 8 * (T ? T : 1), 4 * (d.n_blocks ? d.n_blocks : 1)};
    for (int i = 0; i < BM25X_N_ARRAYS; i++) {
        ptr[i] = p[i];
        bytes[i] = b[i];
    }
}

extern "C" int bm25x_index_get_layout(const bm25x_index *ix, bm25x_index_layout *out) {
    if (!ix || !out) {
        bm25x_set_error("bm25x_index_get_layout: null argument");
        return BM25X_ERR_INVALID;
    }
    out->n_docs = ix->d.n_docs;
    out->n_terms = ix->d.n_terms;
    out->n_postings = ix->d.n_post;
    out->n_postings_padded = ix->d.n_post_pad;
    out->n_blocks = ix->d.n_blocks;
    out->sum_doc_len = ix->sum_len;
    out->k1 = ix->k1;
    out->b = ix->b;
    out->avgdl = ix->avgdl;
    out->device = ix->device;
    layout_arrays(ix, out->dev_ptr, out->bytes);
    return BM25X_OK;
}

extern "C" int bm25x_index_get_derived(const bm25x_index *ix, bm25x_index_derived *out) {
    if (!ix || !out) {
        bm25x_set_error("bm25x_index_get_derived: null argument");
        return BM25X_ERR_INVALID;
    }
    const DeviceIndex &d = ix->d;
    memset(out, 0, sizeof(*out));
    out->pdoc = d.pdoc;
    out->pdoc_bytes = sizeof(uint32_t) * (d.n_post_pad + BM25X_POST_SLACK);
    if (d.champ) {  // a replica has none before its first finalize
        out->champ = d.champ;
        out->champ_bytes = sizeof(Posting) * d.n_champ;
        out->champ_off = d.champ_off;
        out->champ_off_bytes = sizeof(uint64_t) * ((uint64_t)d.n_terms + 1);
        out->n_champ = d.n_champ;
    }
    out->s1f_min = ix->s1f_min;
    out->device = ix->device;
    return BM25X_OK;
}

extern "C" int bm25x_index_alloc_replica(const bm25x_index_layout *like, int device, bm25x_index **out) {
    if (!like || !out) {
        bm25x_set_error("bm25x_index_alloc_replica: null argument");
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        bm25x_set_error("bm25x_index_alloc_replica: CUDA device %d not available; there is no CPU fallback", device);
        return BM25X_ERR_CUDA;
    }
    IndexGuard ix;
    int rc = handle_open("bm25x_index_alloc_replica", device, ix);
    if (rc != BM25X_OK) return rc;
    ix->k1 = like->k1;
    ix->b = like->b;
    ix->avgdl = like->avgdl;
    ix->sum_len = like->sum_doc_len;
    DeviceIndex &d = ix->d;
    d.n_docs = like->n_docs;
    d.n_terms = like->n_terms;
    d.n_post = like->n_postings;
    d.n_post_pad = like->n_postings_padded;
    d.n_blocks = like->n_blocks;
    rc = alloc_arrays(ix.get());
    if (rc == BM25X_OK) *out = ix.release();
    return rc;
}

extern "C" int bm25x_index_finalize_replica(bm25x_index *ix) {
    if (!ix) {
        bm25x_set_error("bm25x_index_finalize_replica: null argument");
        return BM25X_ERR_INVALID;
    }
    BM25X_CUDA_TRY(cudaSetDevice(ix->device));
    // derived data that does not travel: the doc-id-only copy of the postings
    k_extract_docs<<<ix->sm_count * 8, 256>>>(ix->d.post, ix->d.n_post_pad + BM25X_POST_SLACK, ix->d.pdoc);
    BM25X_CUDA_TRY(cudaGetLastError());
    BM25X_CUDA_TRY(cudaDeviceSynchronize());
    ix->h_df.resize(ix->d.n_terms);
    if (ix->d.n_terms)
        BM25X_CUDA_TRY(cudaMemcpy(ix->h_df.data(), ix->d.df, sizeof(uint32_t) * ix->d.n_terms, cudaMemcpyDeviceToHost));
    BM25X_CUDA_TRY(build_champions(ix));  // derived data: built here from the replicated arrays, on every call
    // s1f_min from the replicated arrays
    std::vector<uint8_t> h_fn(ix->d.n_docs);
    float h_s1f[256];
    BM25X_CUDA_TRY(cudaMemcpy(h_fn.data(), ix->d.fieldnorm, ix->d.n_docs, cudaMemcpyDeviceToHost));
    BM25X_CUDA_TRY(cudaMemcpy(h_s1f, ix->d.s1f, sizeof(h_s1f), cudaMemcpyDeviceToHost));
    ix->s1f_min = s1f_min(h_fn.data(), ix->d.n_docs, h_s1f);
    return BM25X_OK;
}

extern "C" int bm25x_index_set_option(bm25x_index *ix, const char *name, int64_t value) {
    if (!ix || !name) {
        bm25x_set_error("bm25x_index_set_option: null argument");
        return BM25X_ERR_INVALID;
    }
    if (strcmp(name, "prune") == 0) {
        ix->prune = value != 0;
        return BM25X_OK;
    }
    if (strcmp(name, "seed") == 0) {  // 2..4-term classes: pools seeded from the champion lists, doc-id-only stream
        ix->seed = value != 0;
        return BM25X_OK;
    }
    if (strcmp(name, "seed_prune_min") == 0) {  // seeded launches: list length from which a skewed query goes to the pruning kernel
        ix->seed_prune_min = value < 0 ? 0u : (value > 0xFFFFFFFFll ? 0xFFFFFFFFu : (uint32_t)value);
        return BM25X_OK;
    }
    if (strcmp(name, "slice_min") == 0) {  // bm25x_search_batch: queries per slice of a pipelined call (0: one piece)
        ix->slice_min = value < 0 ? 0u : (value > 0xFFFFFFFFll ? 0xFFFFFFFFu : (uint32_t)value);
        return BM25X_OK;
    }
    if (strcmp(name, "seed_dense_div") == 0) {  // seeded launches: lists of n_docs / this or more go to the plain kernel (0: never)
        ix->seed_dense_div = value < 0 ? 0u : (value > 0xFFFFFFFFll ? 0xFFFFFFFFu : (uint32_t)value);
        return BM25X_OK;
    }
    if (strcmp(name, "seed_max_terms") == 0) {  // widest term-count class that runs seeded: 4 or 8
        ix->seed_max_terms = value >= 8 ? 8 : 4;
        return BM25X_OK;
    }
    if (strcmp(name, "twophase") == 0) {  // 2..4-term classes: 8-byte postings first, doc ids only once no posting passes alone
        ix->twophase = value != 0;
        return BM25X_OK;
    }
    bm25x_set_error("bm25x_index_set_option: unknown option '%s'", name);
    return BM25X_ERR_INVALID;
}

extern "C" int bm25x_index_get_df(const bm25x_index *ix, uint32_t *df_out) {
    if (!ix || (!df_out && ix->d.n_terms)) {
        bm25x_set_error("bm25x_index_get_df: null argument");
        return BM25X_ERR_INVALID;
    }
    if (ix->h_df.size() != ix->d.n_terms) {
        bm25x_set_error("bm25x_index_get_df: replica not finalized");
        return BM25X_ERR_INVALID;
    }
    memcpy(df_out, ix->h_df.data(), sizeof(uint32_t) * ix->d.n_terms);
    return BM25X_OK;
}

// address_tokens::read (crates/bm25/src/address_tokens.rs:61-98) over the sorted key array.
extern "C" int bm25x_lookup_terms(const bm25x_index *ix, const uint8_t *keys, uint32_t n, uint32_t *out) {
    if (!ix || (!keys && n) || (!out && n)) {
        bm25x_set_error("bm25x_lookup_terms: null argument");
        return BM25X_ERR_INVALID;
    }
    if (ix->h_keys.empty() && ix->d.n_terms) {
        bm25x_set_error("bm25x_lookup_terms: index was created without term keys");
        return BM25X_ERR_INVALID;
    }
    const uint8_t *base = ix->h_keys.data();
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t *key = keys + (size_t)i * 16;
        uint32_t lo = 0, hi = ix->d.n_terms;
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1;
            if (memcmp(base + (size_t)mid * 16, key, 16) < 0) lo = mid + 1;
            else hi = mid;
        }
        out[i] = (lo < ix->d.n_terms && memcmp(base + (size_t)lo * 16, key, 16) == 0) ? lo : BM25X_TERM_MISSING;
    }
    return BM25X_OK;
}
