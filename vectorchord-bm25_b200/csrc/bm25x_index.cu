// bm25x_index.cu — index lifetime: host CSR (the reference's sealed Segment) → flat HBM layout.
//
// Replaces, for the read path, bm25::build → flush (crates/bm25/src/build.rs:22-71,
// crates/bm25/src/flush.rs:40-158): same semantics (N, Σlen → avgdl from exact lengths, per-document
// quantised fieldnorm, 128-posting blocks in (term, doc) order with min/max doc per block, df per
// token) but none of its page / tape / address-tree machinery.  Layout in DESIGN.md §3.
//
// Here: the build core every handle is made by (declared in bm25x_build.h), the CSR builds (one index, document-sharded)
// and the handle API.  The stored-block ingests are in bm25x_blocks.cu, the growing segment in bm25x_growing.cu.
#include <math.h>
#include <omp.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <optional>

#include "bm25x_build.h"

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
uint64_t doc_norms(uint32_t N, const uint32_t *doc_len, const uint8_t *stored_fn, uint64_t stored_sum, uint8_t *fn) {
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

// Stats (bm25x_build.h): the one place the statistics of a handle are computed.
Stats::Stats(uint32_t N, uint64_t sum_len, double avgdl, const uint32_t *df, uint32_t T, double k1, double b)
    : sum_len(sum_len), avgdl(avgdl), s0d(T), s0f(T) {
    for (uint32_t t = 0; t < T; t++) {
        s0d[t] = bm25_s0((double)df[t], (double)N, k1);
        s0f[t] = (float)s0d[t];
    }
    bm25_s1(k1, b, avgdl, s1d);
    for (int f = 0; f < 256; f++) s1f[f] = (float)s1d[f];
}

Stats::Stats(uint32_t N, uint64_t sum_len, const uint32_t *df, uint32_t T, double k1, double b)
    : Stats(N, sum_len, (double)sum_len / (double)N, df, T, k1, b) {}

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

// The refusal for a failed CUDA call of a build step.
int cuda_refusal(const char *who, const char *step, cudaError_t e) {
    bm25x_set_error("%s: %s failed: %s", who, step, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? BM25X_ERR_OOM : BM25X_ERR_CUDA;
}

int check_device(const char *who, int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        bm25x_set_error("%s: CUDA device %d not available (%d devices); there is no CPU fallback", who, device, ndev);
        return BM25X_ERR_CUDA;
    }
    return BM25X_OK;
}

int check_common(const char *who, uint32_t n_docs, const void *doc_len, double k1, double b, int device) {
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

int check_keys(const char *who, const uint8_t *term_key, uint32_t T) {
    if (term_key)
        for (uint32_t t = 1; t < T; t++)
            if (memcmp(term_key + (size_t)(t - 1) * 16, term_key + (size_t)t * 16, 16) >= 0) {
                bm25x_set_error("%s: term_key must be strictly ascending", who);
                return BM25X_ERR_INVALID;
            }
    return BM25X_OK;
}

uint32_t key_ordinal(const uint8_t *keys, uint32_t T, const uint8_t *key) {
    uint32_t lo = 0, hi = T;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (memcmp(keys + (size_t)mid * 16, key, 16) < 0) lo = mid + 1;
        else hi = mid;
    }
    return lo < T && memcmp(keys + (size_t)lo * 16, key, 16) == 0 ? lo : BM25X_TERM_MISSING;
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

// The payload of a document created without one: a synthetic ctid (block hi, block lo, offset) of a 291-tuple page.
void synth_ctid(uint32_t g, uint16_t *out) {
    const uint32_t blkno = g / 291;
    out[0] = (uint16_t)(blkno >> 16);
    out[1] = (uint16_t)(blkno & 0xFFFF);
    out[2] = (uint16_t)(g % 291 + 1);
}

// A handle with everything but the postings, scoring with the `given` statistics (a shard's or a growing segment's: its
// segment's) or, when NULL, its own.  Refusals name bm25x_index_create whichever entry point builds.
int index_begin(const BuildMeta &m, const Stats *given, int device, IndexGuard &ix) {
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
        // of the segment's doc id (a shard's local ids start at doc_base)
        for (uint32_t i = 0; i < N; i++) synth_ctid(m.doc_base + i, &pl[(size_t)i * 3]);
        BM25X_CUDA_TRY(cudaMemcpy(d.payload, pl.data(), sizeof(uint16_t) * pl.size(), cudaMemcpyHostToDevice));
    }
    return BM25X_OK;
}

// After the postings are in place: pad slots, block descriptors, per-term score bounds.
cudaError_t index_finish_device(bm25x_index *ix) {
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
int upload_csr(bm25x_index *ix, const char *who, uint32_t T, uint64_t P, const uint64_t *post_off,
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
    if (sx->eval_df || sx->eval_idf) {
        cudaSetDevice(sx->shards[0]->device);
        cudaFree(sx->eval_df);
        cudaFree(sx->eval_idf);
    }
    for (bm25x_index *ix : sx->shards) bm25x_index_destroy(ix);
    delete sx;
}

// The shard arguments of a document-sharded build, by bm25x_sharded_create's rules and with its messages whichever entry
// point is called: 1..BM25X_MAX_SHARDS shards, at least one document each, explicit bounds strictly ascending from 0 to N.
int check_shard_args(uint32_t N, uint32_t S, const uint32_t *doc_bounds) {
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
std::vector<uint32_t> shard_bounds(const uint32_t *doc_bounds, const std::vector<uint64_t> &cum, uint32_t N,
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

extern "C" void bm25x_index_destroy(bm25x_index *ix) {
    if (!ix) return;
    cudaSetDevice(ix->device);
    if (ix->stream) cudaStreamSynchronize(ix->stream);
    for (void *p : ix->allocs) cudaFree(p);
    cudaFree(ix->key_vocab);
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
    {   // a refill brings another df: bm25x_evaluate_batch rebuilds its idf table from the new one on its next call (the
        // fieldnorm -> length table depends on nothing and stays)
        std::lock_guard<std::mutex> lk(ix->eval_mutex);
        if (ix->eval_idf) {
            ix->allocs.erase(std::find(ix->allocs.begin(), ix->allocs.end(), (void *)ix->eval_idf));
            BM25X_CUDA_TRY(cudaFree(ix->eval_idf));
            ix->eval_idf = nullptr;
        }
    }
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
    for (uint32_t i = 0; i < n; i++) out[i] = key_ordinal(ix->h_keys.data(), ix->d.n_terms, keys + (size_t)i * 16);
    return BM25X_OK;
}
