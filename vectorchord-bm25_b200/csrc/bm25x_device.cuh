// bm25x_device.cuh — device-side building blocks of the search kernel (sm_90a): launch parameters, mbarrier / TMA
// bulk-copy PTX helpers, the two score functions (f32 filter, f64 exact), the tie signature and the warp-private pool.
#pragma once

#include "bm25x_common.h"

// Two-phase launches of the 2..4-term classes (bm25x_search_ring.cuh, RING_SUSPEND then RING_RESUME): what the first
// phase hands over when it suspends a query — the pool entries themselves travel in the query's output rows.
struct ResumeRec {
    double Sk, ub_ne;
    unsigned long long fetched_unused;
    uint32_t rd[4];           // postings consumed per run
    float ne_prefix[4];       // lane t: Σ bounds of the terms pruned before the t-th one
    uint32_t lo, pn, dk, tie_sig, ne_mask, n_ne, ne_list, pad_;
};
static_assert(sizeof(ResumeRec) == 88, "ResumeRec layout");

// One launch = the queries of one term-count class (shared by the translation units of the library).
struct SearchParams {
    const Posting *post;
    const uint32_t *pdoc;               // doc ids of `post` alone, same offsets (RCfg::DOCRING classes stream these)
    const uint64_t *post_off;
    const uint32_t *df;
    const uint64_t *blk_off;
    const uint2 *blk;
    const float *blk_ub;                // [n_blocks] per-block score bound (SummaryTuple.wand_*)
    const float *s0f;
    const double *s0d;
    const double *s1d;
    const float *s1f;
    const uint16_t *payload;
    const double *ubd;                  // per-term upper bound of one posting's exact score
    // two-phase launches: q2[0] = number of suspended queries, q2[1] = the second phase's work counter, q2[2..] = their
    // positions in this launch's query list; resume[position] = the hand-over record
    uint32_t *q2;
    ResumeRec *resume;
    // champion lists (DeviceIndex::champ): seeded launches (RCfg::SEEDED) take their single-term documents from these
    const Posting *champ;
    const uint64_t *champ_off;
    uint32_t seed_dense_div;            // seeded launch: a query with a list of n_docs / this postings or more goes to the plain kernel (0: never)
    uint32_t seed_prune_min;            // seeded launch: a query with a list this long, 8x its shortest one, goes to the pruning kernel
    unsigned long long *fetched;        // Σ postings actually loaded into shared memory (pruning statistics)
    uint8_t *pool_scratch;              // k > 1024: per-warp candidate pools in HBM (k_search_ring, RCfg::POOL_GLOBAL)
    int prune;
    float s1f_min;                      // min over the documents of s1f[fieldnorm]
    uint32_t n_docs;
    // one launch = the queries of one term-count class
    const uint32_t *q_ids;    // original query index
    const uint32_t *q_off;    // [nq+1]
    const uint32_t *q_terms;  // canonical: ascending, distinct, df > 0
    uint32_t nq;
    uint32_t k;
    const uint8_t *allow;
    int *work_counter;
    uint32_t *out_doc;
    float *out_score;
    double *out_score64;
    uint16_t *out_payload;
    uint32_t *out_n;
};

namespace {

constexpr uint32_t INF = BM25X_DOC_INF;

// ---------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + 1-D bulk async copy (TMA)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t addr = smem_u32(bar);
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(addr), "r"(parity)
            : "memory");
        if (!ok) __nanosleep(40);  // do not burn issue slots of the merge warps while waiting
    } while (!ok);
}
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Signature of a single-term document: (run, tf, fieldnorm).  Two documents with the same signature have bit-identical
// exact scores, so "same signature as the current k-th entry and a larger doc id" can be rejected without arithmetic.
constexpr uint32_t SIG_NONE = 0xFFFFFFFFu;
__device__ __forceinline__ uint32_t make_sig(uint32_t j, uint32_t w) {
    return (w >> 27) ? SIG_NONE : ((j << 27) | w);  // tf >= 2^19 does not fit beside the 5-bit run index
}

__device__ __forceinline__ bool key_before(uint64_t ka, uint32_t da, uint64_t kb, uint32_t db) {
    return ka > kb || (ka == kb && da < db);  // score desc, doc asc (scores are > 0: raw f64 bits are monotone)
}

// Cache::evaluate (bm25.rs:355-358) in f32, for the filter only.
__device__ __forceinline__ float score_f32(uint32_t w, float s0, const float *s1f) {
    float tff = (float)(w >> 8);
    float r;  // tf + s1 >= 1: no range guard needed around the approximate reciprocal (1 ulp)
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(tff + s1f[w & 0xFFu]));
    return tff * s0 * r;
}
// Cache::evaluate in f64, bit-exact: (tf * s0) / (tf + s1[fieldnorm]).
__device__ __forceinline__ double score_f64(uint32_t w, double s0, const double *s1d) {
    double tfd = (double)(w >> 8);
    return __ddiv_rn(__dmul_rn(tfd, s0), __dadd_rn(tfd, s1d[w & 0xFFu]));
}

// Warp-private pool: (score bits, doc, signature), unsorted until pool_cut.
template <class C>
struct WPool {
    uint64_t *s;
    uint32_t *d, *g;
};

// Bitonic sort of the warp's pool (n2 = power of two >= n), best first; then keep the best `k`.
template <class C>
__device__ __forceinline__ void wpool_sort(const WPool<C> &pl, int n, int lane) {
    int n2 = 2;
    while (n2 < n) n2 <<= 1;
    for (int i = n + lane; i < n2; i += 32) {
        pl.s[i] = 0;
        pl.d[i] = INF;
        pl.g[i] = SIG_NONE;
    }
    __syncwarp();
    for (int size = 2; size <= n2; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = lane; i < (n2 >> 1); i += 32) {
                int a = 2 * i - (i & (stride - 1));
                int b = a + stride;
                uint64_t ka = pl.s[a], kb = pl.s[b];
                uint32_t da = pl.d[a], db = pl.d[b];
                bool desc = (a & size) == 0;
                bool sw = desc ? key_before(kb, db, ka, da) : key_before(ka, da, kb, db);
                if (sw) {
                    pl.s[a] = kb;
                    pl.s[b] = ka;
                    pl.d[a] = db;
                    pl.d[b] = da;
                    uint32_t ga = pl.g[a];
                    pl.g[a] = pl.g[b];
                    pl.g[b] = ga;
                }
            }
            __syncwarp();
        }
    }
}

struct WFilter {
    bool tv;
    float Flo;   // f32 scores below this cannot reach the top-k
    float ctf;   // lane j: single-term postings of run j pass iff tf >= ctf * s1[fn]   (the same test, solved for tf)
    double Sk;
    uint32_t dk, tie_sig, tie_dk;
};
__device__ __forceinline__ bool wfilter_pass(const WFilter &f, float F, uint32_t sig, uint32_t doc) {
    return F >= f.Flo && !(sig == f.tie_sig && doc > f.tie_dk);
}

}  // namespace
