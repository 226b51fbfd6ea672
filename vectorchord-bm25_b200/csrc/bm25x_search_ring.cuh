// bm25x_search_ring.cuh — kernel v6 (sm_90a): one WARP per query, ring stages + presence map, seeded flavour.
//
// Replaces the per-query cursor walk of bm25::search (crates/bm25/src/search.rs:137-282) for a whole batch: every
// warp of the persistent grid is a complete query engine (lane j owns term j of its query).
//
//   rings     each term ("run") owns a ring of postings in shared memory (the classes of 8+ terms split the warp's ring
//             budget per query in proportion to the terms' df), filled by TMA bulk copies
//             (cp.async.bulk + mbarrier).  A refill appends exactly as many postings as earlier chunks consumed, so
//             every posting crosses L2 → shared memory once (the v5 kernel re-fetched the unconsumed tail of every
//             chunk: 1.66 postings loaded per posting consumed).  A ring is one window, refilled after its chunk from
//             bytes an L2 prefetch issued one round earlier has already pulled into L2.
//   window    chunk = doc window [lo, hi): hi = the smallest "last landed doc" over the runs that still have postings
//             in HBM; each lane binary-searches hi in its run → exact in-window range [rd, e), nothing scanned twice.
//   union     runs are processed in ascending order; run j first TESTS each of its documents against a presence map
//             that holds the marks of runs < j, then MARKS it.  The map is a blocked Bloom filter: a document sets /
//             tests three bits of one 32-bit word (one multiplicative hash; word and bits by shifts of it; a run that
//             tests and marks does both with one atomicOr), cleared per window.  A document held by two runs is
//             therefore always detected by the later run's posting (no false negatives); false alarms (all three bits
//             set by other documents) are about 6 per 1 440-posting chunk of the seeded kernel on C3 (DESIGN.md §4.1).
//   single    a document held by one run only can enter the top-k only if its term frequency passes the threshold:
//             one integer compare per posting (w > wlim_j, wlim_j from the exact threshold solved for tf), plus the
//             tie shortcut (same (run, tf, fieldnorm) signature as the k-th entry ⇒ identical score ⇒ rejected
//             unless the doc id is smaller).
//   verify    detected postings are listed (ballot-compacted) and verified 32 at a time: binary search of the
//             document in the other runs' window ranges, f32 filter score over all holders; the LAST run holding a
//             document emits it (exactly once per document); survivors of the filter are re-scored in f64 in the
//             reference's operation order (Cache::evaluate, bm25.rs:355-358, summed over ascending terms) and enter
//             the warp's pool.
//   dense     windows in which the runs overlap heavily (head terms) are summed in a dense f32 accumulator indexed by
//             doc - lo instead (the window is clamped to the accumulator size: a ring can be consumed partially).
//   pruning   MaxScore-style, as v5 (token-level bounds; non-streamed terms are probed in HBM for candidates).
//
// Flavours (RCfg::FLAVOUR, RingFlavour in bm25x_common.h).  The above is the PLAIN kernel (RING_PLAIN; RING_HANDBACK =
// the same, fed from a device-side query list).  The
// SEEDED kernel (RING_SEEDED; 2..8 terms, k <= 128, no prefilter) takes the documents that hold a single query term from per-term
// champion lists (DeviceIndex::champ: a term's best postings in result order — such a document can only be in the
// top-k if it is among the first k champions of its term).  Its seeds join the candidate list of the doc window they
// fall into and go through the ordinary verification; the stream itself then never tests a posting on its own, so the
// rings hold doc ids only (DeviceIndex::pdoc, 4 B per posting: twice the postings per ring byte, half the HBM bytes),
// posting words are fetched from HBM for the holders of verified documents alone — the ring searches of a verification
// pass only list them in a per-warp hit list, scored (word loads, filter, exact score, pool) up to 32 at a time across
// passes and windows (classes with room for 16 rows or more, RCfg::HITS) — and there is no pruning: queries
// with a dense list or a list much longer than another one are handed back to the plain kernel (RING_HANDBACK launch
// behind it).  Two-phase launches (option "twophase", off by default; 2..4 terms): RING_SUSPEND = the plain kernel,
// which suspends a query once no posting can pass alone, then RING_RESUME = doc-id-only rings that resume it.
//
// Exactness (DESIGN.md §5): the f32 filter only rejects F < Sk·(1-2^-18) and exact-score ties by signature;
// everything else is ranked by (f64 score desc, doc id asc).
#pragma once

#include "bm25x_device.cuh"

namespace {

#ifndef BM25X_RING_LOG_R
#define BM25X_RING_LOG_R -1
#endif
#ifndef BM25X_RING_LOG_S
#define BM25X_RING_LOG_S -1  // log2 of the map bytes; -1: per class (2 KiB of bit cells up to 4 terms, 8 KiB beyond)
#endif
#ifndef BM25X_RING_U
#define BM25X_RING_U 2
#endif
#ifndef BM25X_RING_MAXWARPS
#define BM25X_RING_MAXWARPS 20  // 20 warps = 96 registers per thread.  C3 on H100: 16 warps slower; a cap of 24 still
                                // builds 20 warps of the seeded 3-term class (11 KiB per warp fit 20 times), and 24 real
                                // warps of it (seeds in registers, 80 registers) were 12 % slower (DESIGN.md §7)
#endif
#ifndef BM25X_RING_INIT
#define BM25X_RING_INIT 32
#endif
#ifndef BM25X_RING_DENSE_T
#define BM25X_RING_DENSE_T 48
#endif
#ifndef BM25X_DOCRING_LOG_R
#define BM25X_DOCRING_LOG_R 9  // doc ids per run of a DOCRING class (2 KiB per run, as 256 8-byte postings)
#endif
#ifndef BM25X_DOCRING_G
#define BM25X_DOCRING_G 1  // 16-byte shared loads (4 doc ids) per lane and trip of a DOCRING class
#endif
#ifndef BM25X_DOCRING_TMAX
#define BM25X_DOCRING_TMAX 4  // trips between two compactions of the detected postings of a DOCRING class
#endif
#ifndef BM25X_DOCRING_LOG_S
#define BM25X_DOCRING_LOG_S 11  // log2 of the presence map bytes of a DOCRING class
#endif
#ifndef BM25X_SUSPEND_MIN
#define BM25X_SUSPEND_MIN 4096  // first phase: a query is handed to the doc-id-only phase when at least this many postings remain
#endif
#ifndef BM25X_PRUNE_ALPHA
#define BM25X_PRUNE_ALPHA 0.5  // terms leave the streamed set while the sum of their score bounds stays <= ALPHA · k-th score
#endif

// FLAVOUR_ (a RingFlavour, kept an int so that the kernel names stay plain numbers):
//   RING_PLAIN     one launch answers the query.
//   RING_SUSPEND   two-phase launches of the 2..4-term classes, first phase (8-byte postings in the rings: every posting's
//                  tf / fieldnorm word is at hand while single-term postings can still enter the top-k), which SUSPENDS a
//                  query as soon as no posting can pass alone any more;
//   RING_RESUME    second phase (doc-id-only rings: twice the postings per ring byte, half the bytes from HBM), which
//                  resumes the suspended queries.
//   RING_SEEDED    one seeded launch (2..8 terms).
//   RING_HANDBACK  the plain kernel behind a seeded launch, over the queries it handed back.
template <int M_, int KP_, int FLAVOUR_>
struct RCfg {
    static constexpr int M = M_;    // max live terms (lanes 0..M-1 own the terms)
    static constexpr int FLAVOUR = FLAVOUR_;
    static_assert(FLAVOUR_ == RING_PLAIN || (M_ >= 2 && M_ <= 8 && KP_ <= 256),
                  "flavours other than plain: 2..8 terms, pools in shared memory");
    static_assert((FLAVOUR_ != RING_SUSPEND && FLAVOUR_ != RING_RESUME) || M_ <= 4, "two-phase hand-over record: 4 runs");
    static constexpr int KP = KP_;  // pool capacity (power of two >= k + 32)
    // pools beyond 2048 entries (k > 1024, up to the reference's bm25.limit maximum of 65535, src/index/gucs.rs:37-46)
    // live in HBM: one KP-entry slice of SearchParams::pool_scratch per warp
    static constexpr bool POOL_GLOBAL = KP_ > 2048;
    static constexpr size_t POOL_SMEM = POOL_GLOBAL ? 0 : (size_t)KP_;
    // doc-id-only rings (the resume and seeded flavours): ring element = u32 doc id (SearchParams::pdoc, 4 B per
    // posting: twice the postings per ring byte); the posting word comes from HBM for the few postings that reach the
    // verification
    static constexpr bool DOCRING = FLAVOUR_ == RING_RESUME || FLAVOUR_ == RING_SEEDED;
    // the queries come from the list another launch handed over (SearchParams::q2), not from the batch's work counter
    static constexpr bool FROM_Q2 = FLAVOUR_ == RING_RESUME || FLAVOUR_ == RING_HANDBACK;
    // one SEEDED launch — the documents that hold a single query term come from the terms' champion lists
    // (DeviceIndex::champ) before the stream starts, so the stream (doc ids only) never tests a posting on its own
    // A seeded launch never prunes terms (no single-posting test, no probes: a leaner loop) — queries that would gain
    // from pruning (one list much longer than another) are handed back for the plain kernel (RING_HANDBACK).
    static constexpr bool SEEDED = FLAVOUR_ == RING_SEEDED;
    using RT = typename std::conditional<DOCRING, uint32_t, Posting>::type;  // ring element
    static constexpr uint32_t AL = DOCRING ? 4u : 2u;                        // ring elements per 16 bytes (TMA granularity)
    static constexpr int LOG_R = DOCRING ? BM25X_DOCRING_LOG_R : (BM25X_RING_LOG_R > 0 ? BM25X_RING_LOG_R : (M_ <= 8 ? 8 : 7));
    static constexpr int R = 1 << LOG_R;   // ring postings per run when the M runs share the budget evenly
    // The warp's ring budget (M·R postings) is split per QUERY in proportion to the terms' df (power-of-two rings of
    // 2^LOG_RMIN .. 2^LOG_RMAX postings): head terms next to rare ones get wide windows instead of M equal rings of
    // which the rare terms' stay empty; queries with fewer than M terms use the whole budget.
    static constexpr int BUDGET = M_ * R;
    // Only the classes of 8+ terms size their rings per query (that is where head terms meet rare ones); for 1..4 terms
    // the geometry stays a compile-time constant (M equal rings): runtime masks and bases slow the 3-term loop down.
    static constexpr bool ADAPT = M_ >= 8;
    static constexpr int LOG_RMIN = 6;
    static constexpr int LOG_RMAX = LOG_R + 2 < 10 ? LOG_R + 2 : 10;
    // log2 of the presence map bytes = dense accumulator bytes (unused for one term)
    static constexpr int LOG_S = M_ == 1 ? 8 : (DOCRING && M_ <= 4) ? BM25X_DOCRING_LOG_S : (BM25X_RING_LOG_S > 0 ? BM25X_RING_LOG_S : (M_ <= 4 ? 11 : 13));
    static constexpr uint32_t MAP_BYTES = 1u << LOG_S;
    static constexpr uint32_t ACC_DOCS = MAP_BYTES / 4u;
    static constexpr int U = DOCRING ? BM25X_DOCRING_G : BM25X_RING_U;  // 16-byte shared loads per lane and trip
    static constexpr int E = DOCRING ? 4 : 2;       // postings per 16-byte load
    static constexpr int PL = U * E;                // postings per lane and trip
    static constexpr int TRIP = 32 * PL;            // postings per warp trip
    // trips between two compactions of the detected postings (3: the list stays small enough for a 14th warp per SM)
    static constexpr int TMAX = DOCRING ? BM25X_DOCRING_TMAX : (32 / PL < 3 ? 32 / PL : 3);
    static_assert(PL * TMAX <= 32, "one detection bit per posting slot of a lane between two compactions");
    static constexpr int LCAP = TMAX * TRIP + 64;   // candidate list entries, 16 bits each (verified when > 64 are listed)
    static constexpr int INIT = BM25X_RING_INIT;    // postings per run in the very first load (a threshold exists early)
    static constexpr size_t off_ring = 0;
    static constexpr size_t off_map = off_ring + (size_t)M_ * R * sizeof(RT);
    static constexpr size_t off_pool_s = off_map + (size_t)MAP_BYTES;
    static constexpr size_t off_pool_d = off_pool_s + POOL_SMEM * 8;
    static constexpr size_t off_pool_g = off_pool_d + POOL_SMEM * 4;
    static constexpr size_t off_cand = off_pool_g + POOL_SMEM * 4;
    // seeded launches: the first k champions of the query's terms (doc, w) in shared memory, SST slots per term
    static constexpr uint32_t SST = KP_ <= 64 ? 32u : 128u;
    static constexpr size_t off_seed = (off_cand + (size_t)LCAP * 2 + 7) & ~(size_t)7;
    static constexpr size_t off_hit = off_seed + (SEEDED ? (size_t)M_ * SST * 8 : 0);
    static constexpr size_t off_s1f = 0;  // CTA-shared: 1 KiB table first, then the warps
    static constexpr size_t shared_bytes = 1024;
    static constexpr int MAXW = M_ == 1 ? (BM25X_RING_MAXWARPS > 20 ? BM25X_RING_MAXWARPS : 20) : BM25X_RING_MAXWARPS;
    // seeded launches: the hit list — verified documents waiting for their posting words, scored up to HCAP at a time
    // across windows (struct of arrays: doc ids, then per run the holder's posting index, or the seed's word).  It takes
    // what the 128-byte rounding of the warp's area leaves, up to 32 rows, and never costs a resident warp.  Classes
    // with room for fewer than 16 rows (4 terms at k <= 32, 2 terms at k > 32, 5..8 terms) score each pass's documents
    // right away: a pass can list 32 of them, and a short list would be flushed several times per pass.
    static constexpr int WARPS_NOHIT = (int)((227 * 1024 - shared_bytes) / ((off_hit + 8 + 127) & ~(size_t)127)) > MAXW
                                           ? MAXW
                                           : (int)((227 * 1024 - shared_bytes) / ((off_hit + 8 + 127) & ~(size_t)127));
    static constexpr size_t HIT_ROOM = (((227 * 1024 - shared_bytes) / (WARPS_NOHIT > 0 ? WARPS_NOHIT : 1)) & ~(size_t)127) - (off_hit + 24);
    static constexpr int HROWS = HIT_ROOM / ((M_ + 1) * 4) > 32 ? 32 : (int)(HIT_ROOM / ((M_ + 1) * 4));
    static constexpr bool HITS = SEEDED && HROWS >= 16;
    static constexpr int HCAP = HITS ? HROWS : 0;
    static constexpr size_t off_hst = (off_hit + (size_t)(M_ + 1) * HCAP * 4 + 7) & ~(size_t)7;  // fill state: rows, seed bits
    static constexpr size_t off_bar = off_hst + (HITS ? 8 : 0);
    static constexpr size_t warp_bytes = (off_bar + 8 + 127) & ~(size_t)127;
    static constexpr int WARPS_FIT = (int)((227 * 1024 - shared_bytes) / warp_bytes);
    static constexpr int WARPS = WARPS_FIT > MAXW ? MAXW : WARPS_FIT;
    static_assert(!HITS || WARPS == WARPS_NOHIT, "the hit list costs no resident warp");
    static constexpr size_t total = shared_bytes + warp_bytes * WARPS;
    static constexpr int THREADS = WARPS * 32;
    static_assert(WARPS >= 1, "one warp must fit");
    static_assert(LOG_R <= LOG_RMAX && LOG_R >= LOG_RMIN && M_ <= 32 && MAP_BYTES / 4u <= 32768u && MAP_BYTES % 16u == 0u,
                  "entry format: bit 15 = dense flavour (15-bit doc offset), else 5-bit run | 10-bit ring position");
    static_assert(ACC_DOCS >= 64, "accumulator too small");
};

// -DBM25X_PHASE_PROF (diagnostic build, tools/phase_profile.py): the seeded kernel sums the SM cycles each warp spends in
// every phase of a chunk into g_phase_prof (attribution only: the clock reads cost issue slots and order the code
// around them).  Lane i of a warp accumulates phase i, so the whole profile costs two registers.  Without the flag the
// macros expand to nothing.
enum : int {
    PP_QUERY,    // query start (terms, seeds, first round) and end (final cut, result rows)
    PP_WAIT,     // wait for the refill round (mbar_wait)
    PP_SETUP,    // window limits, boundary searches, dense test
    PP_CLEAR,    // presence map clear
    PP_SEEDS,    // seed listing
    PP_STREAM,   // stream trips (test + mark)
    PP_COMPACT,  // compaction of the detected postings
    PP_VSEARCH,  // verification: ring searches
    PP_VLOAD,    // hit-list flush: wait for the posting-word loads
    PP_VEXACT,   // hit-list append; flush: filter, exact re-score, pool insert
    PP_END,      // chunk end, refill issue
    PP_PHASES,
    PP_CHUNKS = PP_PHASES,  // counters after the phases: chunks, listed candidates, hits (candidates another run confirms,
    PP_CANDS,               // or seeds no other run holds), flushes of the hit list and the rows they scored
    PP_HITS,
    PP_FLUSHES,
    PP_ROWS,
    PP_SLOTS
};
#ifdef BM25X_PHASE_PROF
__device__ unsigned long long g_phase_prof[PP_SLOTS];
#define PP_MARK(ph)                                                \
    do {                                                           \
        if constexpr (C::SEEDED) {                                 \
            const uint32_t pp_now_ = (uint32_t)clock();            \
            if (lane == (ph)) pp_acc += pp_now_ - pp_t;            \
            pp_t = pp_now_;                                        \
        }                                                          \
    } while (0)
#define PP_COUNT(slot, n)                                          \
    do {                                                           \
        if constexpr (C::SEEDED) {                                 \
            const uint32_t pp_n_ = (n); /* every lane takes part */ \
            if (lane == (slot)) pp_acc += pp_n_;                   \
        }                                                          \
    } while (0)
// the clock is read after the loaded words are consumed, so that the wait lands in PP_VLOAD
#define PP_CONSUME(a, b)                                                                      \
    do {                                                                                      \
        if constexpr (C::SEEDED) {                                                            \
            uint32_t pp_x_;                                                                   \
            asm volatile("xor.b32 %0, %1, %2;" : "=r"(pp_x_) : "r"(a), "r"(b));               \
        }                                                                                     \
    } while (0)
#else
#define PP_MARK(ph) do {} while (0)
#define PP_COUNT(slot, n) do {} while (0)
#define PP_CONSUME(a, b) do {} while (0)
#endif

// Presence map: the 32-bit cell word of a document (its word index) and the THREE bits it sets / tests there (a blocked
// Bloom filter: one shared-memory atomicOr or load per posting; false alarms ~ fill^3).  Multiplicative hash; the slot
// is its top log2(cells) bits (the high half of hash × cells of a power-of-two map, one instruction instead of IMAD.HI +
// mask), the second bit comes from its low 5 bits, the third from the next 5.  The bit shifts wrap (SHF.L.W): 1 << x
// takes x's low 5 bits, no mask needed.
template <class C>
__device__ __forceinline__ uint32_t map_word(uint32_t doc, uint32_t &msk) {
    static_assert((C::MAP_BYTES & (C::MAP_BYTES - 1u)) == 0u, "the presence map is a power of two bytes");
    constexpr int LOG_CELLS = 31 - __builtin_clz(C::MAP_BYTES * 8u);
    const uint32_t hsh = doc * 0x9E3779B1u;
    const uint32_t slot = hsh >> (32 - LOG_CELLS);
    uint32_t word;
    // (a shift the compiler cannot merge with the caller's ×4 into shift + mask + add: one IMAD forms the address)
    asm("shr.b32 %0, %1, %2;" : "=r"(word) : "r"(hsh), "n"(32 - LOG_CELLS + 5));
    msk = __funnelshift_l(0u, 1u, slot);
    msk |= __funnelshift_l(0u, 1u, hsh) | __funnelshift_l(0u, 1u, hsh >> 5);
    return word;
}
// lower_bound of `doc` in ring positions [a, e) (posting indices of the term; the ring holds index i at i & RM).
// Fixed LOG_R + 1 power-of-two steps, no data-dependent branch: every lane of a verification pass searches the same run,
// and independent searches interleave (the while-loop form costs several times the instructions per search).
__device__ __forceinline__ uint32_t ring_doc(const Posting *rg, uint32_t pos) { return rg[pos].doc; }
__device__ __forceinline__ uint32_t ring_doc(const uint32_t *rg, uint32_t pos) { return rg[pos]; }
template <class C, int TOP = C::LOG_RMAX>
__device__ __forceinline__ uint32_t ring_lower_bound(const typename C::RT *rg, uint32_t mask, uint32_t a, uint32_t e,
                                                     uint32_t doc) {
    uint32_t pos = a;  // every posting before pos is < doc
#pragma unroll
    for (int s = TOP; s >= 0; --s) {
        const uint32_t probe = pos + (1u << s);
        if (probe <= e && ring_doc(rg, (probe - 1u) & mask) < doc) pos = probe;
    }
    return pos;
}
// posting word of `doc` in [a, e), 0 when absent (8-byte rings)
template <class C, int TOP = C::LOG_RMAX>
__device__ __forceinline__ uint32_t ring_find(const Posting *rg, uint32_t mask, uint32_t a, uint32_t e, uint32_t doc) {
    const uint32_t l = ring_lower_bound<C, TOP>(rg, mask, a, e, doc);
    if (l < e) {
        const Posting v = rg[l & mask];
        if (v.doc == doc) return v.w;
    }
    return 0u;
}

// posting index of `doc` in [a, e), INF when absent (doc-id-only rings: the posting word is fetched by the caller, so that
// the loads of all holders of a candidate are in flight together)
template <class C, int TOP = C::LOG_RMAX>
__device__ __forceinline__ uint32_t ring_find_pos(const typename C::RT *rg, uint32_t mask, uint32_t a, uint32_t e, uint32_t doc) {
    const uint32_t l = ring_lower_bound<C, TOP>(rg, mask, a, e, doc);
    return (l < e && ring_doc(rg, l & mask) == doc) ? l : INF;
}

// ---- probes of a term that is not streamed any more (candidates only; replaces Cursor::seek_block / seek of the
// reference's parked cursors, search.rs:412-466): block table first (SummaryTuple.{min,max}_document_id), then inside
// the 128-posting block.  `steps` counts the table entries / postings read (pruning statistics).
// Returns l = 1 + index of the last block whose first document is <= doc (0: doc lies before the first block).
__device__ __forceinline__ uint32_t probe_block(const SearchParams &p, uint64_t bbase, uint32_t nb, uint32_t doc,
                                                uint32_t &steps) {
    uint32_t l = 0, r = nb;
    while (l < r) {
        const uint32_t mid = (l + r) >> 1;
        if (__ldg(&p.blk[bbase + mid].x) <= doc) l = mid + 1;
        else r = mid;
        steps++;
    }
    return l;
}
__device__ __forceinline__ uint32_t probe_in_block(const SearchParams &p, uint64_t pbase, uint32_t dfj, uint32_t block,
                                                   uint32_t doc, uint32_t &steps) {
    const uint32_t s = block * BM25X_BLOCK, e = min(s + BM25X_BLOCK, dfj);
    const Posting *pp = p.post + pbase;
    uint32_t l = s, r = e;
    while (l < r) {
        const uint32_t mid = (l + r) >> 1;
        if (__ldg(&pp[mid].doc) < doc) l = mid + 1;
        else r = mid;
        steps++;
    }
    if (l < e) {
        const Posting v = pp[l];
        if (v.doc == doc) return v.w;
    }
    return 0u;
}

template <class C>
__global__ void __launch_bounds__(C::THREADS, 1) k_search_ring(const __grid_constant__ SearchParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr uint32_t FULL = 0xFFFFFFFFu;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    float *s1f = (float *)(smem + C::off_s1f);
    for (int i = threadIdx.x; i < 256; i += C::THREADS) s1f[i] = p.s1f[i];
    uint8_t *ws = smem + C::shared_bytes + C::warp_bytes * wid;
    using RT = typename C::RT;
    RT *rings = (RT *)(ws + C::off_ring);
    uint8_t *map = ws + C::off_map;
    WPool<C> pl;
    if (C::POOL_GLOBAL) {
        uint8_t *slice = p.pool_scratch + ((size_t)blockIdx.x * C::WARPS + wid) * ((size_t)C::KP * 16);
        pl.s = (uint64_t *)slice;
        pl.d = (uint32_t *)(slice + (size_t)C::KP * 8);
        pl.g = (uint32_t *)(slice + (size_t)C::KP * 12);
    } else {
        pl.s = (uint64_t *)(ws + C::off_pool_s);
        pl.d = (uint32_t *)(ws + C::off_pool_d);
        pl.g = (uint32_t *)(ws + C::off_pool_g);
    }
    uint16_t *cand = (uint16_t *)(ws + C::off_cand);
    uint64_t *bar = (uint64_t *)(ws + C::off_bar);
    if (lane == 0) {
        mbar_init(bar, 1);
        mbar_fence_init();
        if constexpr (C::HITS) *(uint2 *)(ws + C::off_hst) = make_uint2(0u, 0u);  // the hit list starts empty (every query ends drained)
    }
    if (C::M > 1)
        for (int i = lane; i < (int)(C::MAP_BYTES / 16u); i += 32) ((uint4 *)map)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    const uint32_t k = p.k;
    const double kEps = 1.0 / 262144.0;
    const float s1min = p.s1f_min;
    uint32_t parity = 0;  // mbarrier phase parity
#ifdef BM25X_PHASE_PROF
    uint32_t pp_acc = 0u, pp_t = (uint32_t)clock();  // lane i: cycles of phase i (or counter i) of the current query
#endif

    for (;;) {
        int qi = 0;
        if constexpr (C::FROM_Q2) {  // the queries another launch handed over (suspended / handed back), in that order
            if (lane == 0) {
                const uint32_t i = atomicAdd(&p.q2[1], 1u);
                qi = i < p.q2[0] ? (int)p.q2[2u + i] : -1;
            }
            qi = __shfl_sync(FULL, qi, 0);
            if (qi < 0) break;
        } else {
            if (lane == 0) qi = atomicAdd(p.work_counter, 1);
            qi = __shfl_sync(FULL, qi, 0);
            if (qi >= (int)p.nq) break;
        }
        const uint32_t qid = p.q_ids[qi];
        const uint32_t t0q = p.q_off[qi];
        const uint32_t m_total = p.q_off[qi + 1] - t0q;
        // More than 32 terms (lane j = term j holds 32): TWO passes over term groups — the host puts the 32 rarest terms
        // first.  Pass 0 streams group 0 and probes group 1 for its candidates; pass 1 streams group 1 and owns exactly the
        // documents that hold no group-0 term.  Every document is emitted once, with its full score; pool and threshold
        // span the passes.
        const bool mp = C::M == 32 && m_total > 32u;
        if constexpr (C::SEEDED) {
            // The seeded kernel is the kernel of SPARSE lists.  A query goes back to the plain kernel (8-byte postings: dense
            // windows sum tf / fieldnorm words straight from the rings; MaxScore pruning) when one of its lists is dense
            // (>= n_docs / seed_dense_div postings: its windows overlap the other runs') or much longer than another one
            // (head term next to rare ones: pruning pays).
            uint32_t dfl = 0u;
            if (lane < (int)m_total) dfl = p.df[p.q_terms[t0q + lane]];
            const uint32_t mx = __reduce_max_sync(FULL, dfl);
            const uint32_t mn = __reduce_min_sync(FULL, lane < (int)m_total ? dfl : 0xFFFFFFFFu);
            if ((p.prune && mx >= p.seed_prune_min && mx / 8u >= mn) || (p.seed_dense_div && mx >= p.n_docs / p.seed_dense_div + 1u)) {
                if (lane == 0) {
                    const uint32_t at = atomicAdd(&p.q2[0], 1u);
                    p.q2[2u + at] = (uint32_t)qi;
                }
                continue;
            }
        }
        // postings fetched by this lane (seeded launches: one term's list, < 2^32 — a register less; summed in 64 bits at query end)
        typename std::conditional<C::SEEDED, uint32_t, unsigned long long>::type fetched = 0;
        uint32_t probe_steps = 0;
        // per-query pool / threshold state (warp-uniform registers)
        int pn = 0;
        WFilter f;
        f.tv = false;
        f.Flo = -1.f;
        f.Sk = 0.0;
        f.dk = INF;
        f.tie_sig = SIG_NONE;
        f.tie_dk = INF;
        f.ctf = 0.f;
        bool suspended = false;  // first phase: the query goes on in the second phase
        for (int pass = 0; pass < (mp ? 2 : 1); ++pass) {
        const uint32_t t0 = t0q + (pass ? 32u : 0u);
        const uint32_t m = mp ? (pass ? m_total - 32u : 32u) : m_total;
        const uint32_t obase = t0q + (pass ? 0u : 32u);          // the other group (probed, never streamed in this pass)
        const uint32_t on = mp ? (pass ? 32u : m_total - 32u) : (m_total & 0u);  // (& 0: keeps "on" a runtime zero)
        double ub_oth = 0.0;  // pass 0: Σ score bounds of the other group's terms (they can add to any candidate)
        if (mp && pass == 0) {
            double ub = lane < (int)on ? p.ubd[p.q_terms[obase + lane]] : 0.0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ub += __shfl_xor_sync(FULL, ub, o);
            ub_oth = ub * (1.0 + 1.0e-12);
        }
        // ---- query terms: lane j < m (TokenTuple of term j: df, postings, score constants) ----
        uint32_t dfj = 0, dfpad = 0, nbj = 0;
        uint64_t pbase = 0, bbase = 0;
        float s0f = 0.f;
        double s0d = 0.0, ubd = 0.0;
        if (lane < (int)m) {
            const uint32_t term = p.q_terms[t0 + lane];
            dfj = p.df[term];
            dfpad = (dfj + C::AL - 1u) & ~(C::AL - 1u);  // whole 16-byte pieces (the lists are padded to 4 postings in HBM)
            pbase = p.post_off[term];
            bbase = p.blk_off[term];
            nbj = (dfj + BM25X_BLOCK - 1) / BM25X_BLOCK;
            s0f = p.s0f[term];
            s0d = p.s0d[term];
            ubd = p.ubd[term];
        }
        // ---- ring sizes: ∝ df over the streamed terms, powers of two, Σ <= BUDGET (lane j: 2^rlog postings at
        // rings + rbase).  Called at query start and again whenever terms leave the streamed set (their rings go back to
        // the budget).
        uint32_t rlog = 0, rbase = 0, rsize = 2u, rmask = 1u;
        bool small_rings = true;  // every ring <= 2^LOG_R postings: searches need LOG_R + 1 steps only
        RT *myring = rings;
        auto alloc_rings = [&](uint32_t streamed) {
            if constexpr (!C::ADAPT) {  // M equal rings at fixed places
                rlog = C::LOG_R;
                rbase = (uint32_t)(lane < C::M ? lane : 0) * C::R;
                rsize = C::R;
                rmask = C::R - 1u;
                myring = rings + rbase;
                small_rings = true;
                return;
            }
            const bool mine = lane < (int)m && ((streamed >> lane) & 1u);
            unsigned long long sumdf = mine ? dfj : 0u;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sumdf += __shfl_xor_sync(FULL, sumdf, o);
            uint32_t size = 0;
            rlog = 0;
            {
                // share of the budget, as a power of two: rounded to the NEAREST one when all of these fit, else down
                uint32_t lo2 = 0, near2 = 0;
                if (mine) {
                    const uint32_t share = (uint32_t)(((unsigned long long)C::BUDGET * dfj) / sumdf);
                    lo2 = share > 1u ? 31u - (uint32_t)__clz(share) : 0u;
                    near2 = lo2 + ((unsigned long long)share * share >= (2ull << (2u * lo2)) ? 1u : 0u);  // share >= √2·2^lo2
                    lo2 = min(max(lo2, (uint32_t)C::LOG_RMIN), (uint32_t)C::LOG_RMAX);
                    near2 = min(max(near2, (uint32_t)C::LOG_RMIN), (uint32_t)C::LOG_RMAX);
                    while (lo2 > (uint32_t)C::LOG_RMIN && (1u << (lo2 - 1u)) >= dfpad) lo2--;  // no larger than the list
                    while (near2 > (uint32_t)C::LOG_RMIN && (1u << (near2 - 1u)) >= dfpad) near2--;
                }
                const bool fits = __reduce_add_sync(FULL, mine ? 1u << near2 : 0u) <= (uint32_t)C::BUDGET;
                if (mine) {
                    rlog = fits ? near2 : lo2;
                    size = 1u << rlog;
                }
            }
            uint32_t used = __reduce_add_sync(FULL, size);
            while (used > (uint32_t)C::BUDGET) {  // the minimum sizes of many rare terms can overshoot: halve the largest ring
                const uint32_t big = __reduce_max_sync(FULL, size);
                const uint32_t who = __ballot_sync(FULL, size == big);
                if (lane == __ffs(who) - 1) {
                    rlog--;
                    size >>= 1;
                }
                used -= big >> 1;
            }
            // the rest of the budget: double EVERY ring that can still grow, as long as all of them fit (keeps the
            // proportions: equal terms keep equal rings)
            for (;;) {
                const bool can = mine && rlog < (uint32_t)C::LOG_RMAX && size < dfpad;
                const uint32_t extra = __reduce_add_sync(FULL, can ? size : 0u);
                if (extra == 0u || used + extra > (uint32_t)C::BUDGET) break;
                if (can) {
                    rlog++;
                    size <<= 1;
                }
                used += extra;
            }
            uint32_t incl = size;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(FULL, incl, o);
                if (lane >= o) incl += v;
            }
            rbase = incl - size;
            rsize = mine ? size : 2u;
            rmask = rsize - 1u;
            myring = rings + rbase;
            small_rings = __reduce_max_sync(FULL, rlog) <= (uint32_t)C::LOG_R;
        };
        alloc_rings(FULL);
        // ring geometry of run i (warp-uniform i)
        auto ring_base = [&](int i) -> uint32_t { return C::ADAPT ? __shfl_sync(FULL, rbase, i) : (uint32_t)i * C::R; };
        auto ring_mask = [&](int i) -> uint32_t { return C::ADAPT ? __shfl_sync(FULL, rmask, i) : (uint32_t)C::R - 1u; };
        uint32_t rd = 0, wr = 0;  // my run: postings [0, rd) consumed, [rd, wr) in the ring (wr: landed at the next wait)
        uint32_t lo = 0;          // every posting with doc < lo has been consumed
        // MaxScore pruning (warp-uniform): terms in ne_mask are no longer streamed; ub_ne = Σ of their score bounds
        uint32_t ne_mask = 0u;
        double ub_ne = 0.0;
        uint32_t ne_list = 0u;     // the pruned terms in the order they left (ascending bound), 4 bits each (classes <= 8 terms)
        int n_ne = 0;
        float ne_prefix_f = 0.f;   // lane t: Σ bounds of the terms pruned before the t-th one, rounded up
        float FloT = -1.f;         // filter threshold on the score over ALL terms (f.Flo: over the streamed terms only)
        bool thr_new = false;     // the threshold moved since the pruned set was last reconsidered
        uint32_t wlim = C::SEEDED ? 0xFFFFFFFFu : 255u;  // lane j: single-term postings of run j can pass only if w > wlim  (tf >= 1: all)
        uint32_t tiew = 0xFFFFFFFFu;  // lane j: posting word of the tie signature when it belongs to run j

        // f32 filter constants from (Sk, tie signature, pruned set)
        auto refresh_filter = [&]() {
            f.tie_dk = (f.tie_sig != SIG_NONE && ne_mask == 0u && !mp) ? f.dk : INF;  // pruned / probed terms: no tie shortcut
            const double flo = f.Sk * (1.0 - kEps) - ub_ne - ub_oth;
            f.Flo = __double2float_rd(flo);
            FloT = __double2float_rd(f.Sk * (1.0 - kEps));
            // F = s0·tf/(tf+s1) >= flo  ⇔  tf >= flo/(s0-flo)·s1  (s0 > flo), never when s0 <= flo.  Solved in f64
            // from the exact s0, shrunk by 2^-20 to stay conservative in f32.
            f.ctf = __int_as_float(0x7f800000);  // +inf
            if (lane < (int)m && s0d > flo) f.ctf = __double2float_rd(flo / (s0d - flo) * (1.0 - 1.0 / 1048576.0));
            // one-compare version for the hot loop: tf >= ctf·s1[fn] implies tf >= fl(ctf · min s1) (rounding is monotone),
            // and tf is an integer: tf >= ceil(that).  (floor would let every tf = 1 posting of a term whose best
            // single-term score is just below the threshold through to the verification.)
            uint32_t tfmin = 0x1000000u;
            if (f.ctf < 3.0e38f) {
                const float t = ceilf(f.ctf * s1min);
                tfmin = t < 16777216.f ? (t > 1.f ? (uint32_t)t : 1u) : 0x1000000u;
            }
            wlim = tfmin >= 0x1000000u ? 0xFFFFFFFFu : (tfmin << 8) - 1u;
            // the term's best posting (its token-level bound) stays below the threshold: no posting of this run can
            // enter alone, the hot loop drops the single-term test altogether
            if (lane < (int)m && ubd < flo) wlim = 0xFFFFFFFFu;
            tiew = (f.tie_dk != INF && (f.tie_sig >> 27) == (uint32_t)lane) ? (f.tie_sig & 0x07FFFFFFu) : 0xFFFFFFFFu;
            if constexpr (C::SEEDED) {  // single-term documents come from the champion lists: the stream lists no posting on its own
                wlim = 0xFFFFFFFFu;
                tiew = 0xFFFFFFFFu;
            }
        };
        // cut the pool back to k and refresh the threshold (Results::push / threshold, search.rs:284-314)
        auto pool_cut = [&]() {
            wpool_sort<C>(pl, pn, lane);
            if (pn > (int)k) pn = (int)k;
            if (pn == (int)k) {
                f.Sk = __longlong_as_double((long long)pl.s[k - 1]);
                f.dk = pl.d[k - 1];
                f.tie_sig = pl.g[k - 1];
                f.tv = true;
                thr_new = true;
                refresh_filter();
            }
        };
        // exact score of a filtered document from its holders' posting words, in the reference's operation order
        // (Cache::evaluate, bm25.rs:355-358, summed over ascending terms)
        auto exact_sum = [&](bool keep, const uint32_t (&wv)[C::M], uint32_t &cnt_all) -> double {
            double Sx = 0.0;
#pragma unroll
            for (int i = 0; i < C::M; ++i)
                if (i < (int)m) {
                    const double s0 = __shfl_sync(FULL, s0d, i);
                    if (keep && wv[i]) {
                        Sx = __dadd_rn(Sx, score_f64(wv[i], s0, p.s1d));
                        cnt_all++;
                    }
                }
            return Sx;
        };
        // a re-scored document enters the pool when it beats the k-th entry so far (score desc, doc asc)
        auto pool_insert = [&](bool keep, double Sx, uint32_t doc, uint32_t g) {
            keep = keep && (!f.tv || Sx > f.Sk || (Sx == f.Sk && doc < f.dk));
            const uint32_t mk = __ballot_sync(FULL, keep);
            if (keep) {
                const int idx = pn + __popc(mk & lt_mask);
                pl.s[idx] = (uint64_t)__double_as_longlong(Sx);
                pl.d[idx] = doc;
                pl.g[idx] = g;
            }
            pn += __popc(mk);
            __syncwarp();
            // Re-sorting a large pool is expensive (bitonic sort of KP entries): once a threshold exists,
            // the big pool is cut only when it is about to overflow.
            const bool lazy = C::KP > 128 && f.tv;
            if (pn > C::KP - 32 || (!lazy && pn >= (int)k + 32)) pool_cut();
        };

        // ---- seeded launches: the hit list.  The ring searches of a verification pass decide which documents are
        // live (every holder found, the last streamed holder emits, a seed only when no other run holds it, a streamed
        // document only when two or more do); a live document needs no ring after that, so it waits here as a row (doc
        // id; per run the holder's posting index relative to pbase, INF when the run does not hold it — or, for a seed,
        // its posting word from the seed table and 0 elsewhere) and is scored with up to HCAP - 1 others, one row per
        // lane: one DRAM latency for all their word loads, one filter / exact / pool-insert chain.  Deferring a document
        // only lets the threshold it meets be lower (DESIGN.md §5).  The list's fill state (rows; bit r: row r is a
        // seed) sits beside it in shared memory, not in registers held through the chunk loop.
        auto hit_flush = [&](uint32_t hn, uint32_t hseed) {
            const uint32_t *hl = (const uint32_t *)(ws + C::off_hit);
            __syncwarp();  // every lane's rows are visible
            PP_COUNT(PP_FLUSHES, 1u);
            PP_COUNT(PP_ROWS, hn);
            const bool has = lane < (int)hn;
            const bool sd = (hseed >> lane) & 1u;
            const uint32_t doc = has ? hl[lane] : 0u;
            uint32_t wv[C::M];
#pragma unroll
            for (int i = 0; i < C::M; ++i) {
                const uint32_t v = has ? hl[(i + 1) * C::HCAP + lane] : INF;
                const uint64_t pbi = __shfl_sync(FULL, pbase, i);
                wv[i] = sd ? v : (v != INF ? __ldg(&(p.post + pbi)[v].w) : 0u);
            }
#pragma unroll
            for (int i = 0; i < C::M; ++i) PP_CONSUME(wv[i], wv[0]);
            PP_MARK(PP_VLOAD);
            float F = 0.f;
            uint32_t cnt = 0, sig = SIG_NONE;
#pragma unroll
            for (int i = 0; i < C::M; ++i) {
                const float s0 = __shfl_sync(FULL, s0f, i);
                if (wv[i]) {
                    F += score_f32(wv[i], s0, s1f);
                    cnt++;
                    sig = make_sig(i, wv[i]);
                }
            }
            bool keep = has && wfilter_pass(f, F, cnt == 1 ? sig : SIG_NONE, doc);
            if (keep && p.allow && !((p.allow[doc >> 3] >> (doc & 7u)) & 1u)) keep = false;
            if (__any_sync(FULL, keep)) {
                uint32_t cnt_all = 0;
                const double Sx = exact_sum(keep, wv, cnt_all);
                pool_insert(keep, Sx, doc, cnt_all == 1 ? sig : SIG_NONE);
            }
            __syncwarp();  // every lane has read its row before the list fills again
            PP_MARK(PP_VEXACT);
        };
        // Before a pass's searches: flush when its c candidates might not fit.  A pass holds at most HCAP candidates,
        // so its rows always fit after this, and no search result is live across a flush.
        auto hit_room = [&](uint32_t c) {
            uint32_t *hst = (uint32_t *)(ws + C::off_hst);
            const uint32_t hn = hst[0];
            if (hn != 0u && hn + c > (uint32_t)C::HCAP) {
                hit_flush(hn, hst[1]);
                if (lane == 0) hst[0] = hst[1] = 0u;
                __syncwarp();
            }
        };
        // append the rows of one verification pass (`row`: this lane's document is live; hv: its per-run values)
        auto hit_append = [&](bool row, uint32_t doc, bool sd, const uint32_t (&hv)[C::M]) {
            uint32_t *hl = (uint32_t *)(ws + C::off_hit);
            uint32_t *hst = (uint32_t *)(ws + C::off_hst);
            const uint32_t mk = __ballot_sync(FULL, row);
            if (!mk) return;
            const uint32_t hn = hst[0], r = hn + __popc(mk & lt_mask);
            if (row) {
                hl[r] = doc;
#pragma unroll
                for (int i = 0; i < C::M; ++i) hl[(i + 1) * C::HCAP + r] = hv[i];
            }
            const uint32_t hseed = hst[1] | __reduce_or_sync(FULL, row && sd ? 1u << r : 0u);
            __syncwarp();
            if (lane == 0) {
                hst[0] = hn + __popc(mk);
                hst[1] = hseed;
            }
            __syncwarp();
        };
        // the rows of the last windows, before the final cut
        auto hit_drain = [&]() {
            uint32_t *hst = (uint32_t *)(ws + C::off_hst);
            const uint32_t hn = hst[0];
            if (hn) {
                PP_MARK(PP_QUERY);
                hit_flush(hn, hst[1]);
                if (lane == 0) hst[0] = hst[1] = 0u;
                __syncwarp();
            }
        };

        if (pass && f.tv) {  // second pass: the threshold of the first one, solved for this group's terms
            thr_new = true;
            refresh_filter();
        }

        // one refill round: lane j appends n postings (a multiple of AL = whole 16-byte pieces) to its ring
        auto issue_round = [&](uint32_t n) -> bool {
            const uint32_t total = __reduce_add_sync(FULL, n);
            if (total == 0u) return false;
            // the freed ring slots were last read through the generic proxy by this warp: order those reads before the
            // async-proxy writes
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive_expect_tx(bar, total * (uint32_t)sizeof(RT));
            __syncwarp();
            if (n > 0) {
                const uint32_t off = wr & rmask;
                const uint32_t n1 = min(n, rsize - off);
                const RT *src;
                if constexpr (C::DOCRING) src = p.pdoc + pbase + wr;
                else src = p.post + pbase + wr;
                tma_load_1d(myring + off, src, n1 * (uint32_t)sizeof(RT), bar);
                if (n > n1) tma_load_1d(myring, src + n1, (n - n1) * (uint32_t)sizeof(RT), bar);
                fetched += min(wr + n, dfj) - min(wr, dfj);  // the pad slots of a list are not postings
                wr += n;
            }
            return true;
        };

        bool inflight;
        if constexpr (C::FLAVOUR == RING_RESUME) {
            // ---- resume: cursors, threshold, pruned set from the record; the pool entries from the query's output rows ----
            const ResumeRec *rec = p.resume + qi;
            const size_t ob = (size_t)qid * k;
            pn = (int)rec->pn;
            for (int i = lane; i < pn; i += 32) {
                pl.s[i] = (uint64_t)__double_as_longlong(p.out_score64[ob + i]);
                pl.d[i] = p.out_doc[ob + i];
                pl.g[i] = __float_as_uint(p.out_score[ob + i]);
            }
            if (lane < (int)m) rd = rec->rd[lane];
            if (lane < 4) ne_prefix_f = rec->ne_prefix[lane];
            lo = rec->lo;
            f.tv = true;
            f.Sk = rec->Sk;
            f.dk = rec->dk;
            f.tie_sig = rec->tie_sig;
            ne_mask = rec->ne_mask;
            n_ne = (int)rec->n_ne;
            ne_list = rec->ne_list;
            ub_ne = rec->ub_ne;
            thr_new = true;
            refresh_filter();
            __syncwarp();
            wr = rd & ~(C::AL - 1u);
            inflight = issue_round(lane < (int)m && !((ne_mask >> lane) & 1u) ? min(rsize, dfpad - wr) : 0u);
        } else {
            // (a seeded launch needs no early threshold: whole rings from the start)
            inflight = issue_round(lane < (int)m ? min(dfpad, C::SEEDED ? rsize : (uint32_t)C::INIT) : 0u);
        }
        // ---- seeds: a document that holds ONE query term can only be in the top-k if it is among the first k champions
        // of that term (DeviceIndex::champ: every posting ranked before it in (single-term score desc, doc asc) belongs
        // to a document that beats it).  The first min(k, df) champions of every term are the query's seeds; each is
        // handed to the verification of the doc window it falls into (the rings then hold every other run's postings of
        // that window): a seed no other term holds enters the pool with its exact score, the others are left to the
        // stream, which finds every document held by two terms.  The stream itself never tests a posting on its own.
        uint32_t ncj = 0u;    // lane j: seeds of term j
        uint64_t coff = 0ull;  // lane j: its champion list
        [[maybe_unused]] Posting *seeds = nullptr;
        if constexpr (C::SEEDED) {
            if (lane < (int)m) {
                ncj = min(dfj, min(k, (uint32_t)BM25X_CHAMP_L));
                coff = p.champ_off[p.q_terms[t0 + lane]];
            }
            seeds = (Posting *)(ws + C::off_seed);
#pragma unroll
            for (int jj = 0; jj < C::M; ++jj) {
                const uint32_t nj = __shfl_sync(FULL, ncj, jj);
                const uint64_t cj = __shfl_sync(FULL, coff, jj);
                for (uint32_t r = (uint32_t)lane; r < C::SST && r < ((k + 31u) & ~31u); r += 32) {
                    Posting v;
                    v.doc = INF;  // slots beyond the list: never inside a window
                    v.w = 0u;
                    if (r < nj) v = p.champ[cj + r];
                    seeds[jj * C::SST + r] = v;
                }
            }
            __syncwarp();
        }
        PP_MARK(PP_QUERY);
        for (;;) {
            // ---- chunk boundary: the outstanding round has landed ----
            if (inflight) {
                mbar_wait(bar, parity);
                parity ^= 1u;
            }
            PP_MARK(PP_WAIT);
            PP_COUNT(PP_CHUNKS, 1u);
            // MaxScore (the reference's WAND pivot rule, search.rs:152-169, applied to whole terms): the terms with the
            // smallest score bounds leave the streamed set while the sum of their bounds (plus ub_oth) stays <= ALPHA · k-th
            // score.  A document holding only such terms cannot enter; for the others the bound is added back in the filter and
            // the exact contributions are probed at verification — best bound first, giving up on a document as soon as
            // the block-level bound (SummaryTuple.wand_*, search.rs:193-203) of the probed term plus the bounds of the
            // terms still to probe cannot lift it over the threshold.
            // Only at chunk boundaries: inside a chunk the "last holder emits" rule relies on a fixed streamed set.
            if (!C::SEEDED && p.prune && thr_new) {
                thr_new = false;
                bool changed = false;
                for (;;) {
                    const bool ess = lane < (int)m && !((ne_mask >> lane) & 1u);
                    unsigned long long key = ess ? (unsigned long long)__double_as_longlong(ubd) : ~0ull;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const unsigned long long other = __shfl_xor_sync(FULL, key, o);
                        key = other < key ? other : key;
                    }
                    const uint32_t who = __ballot_sync(FULL, ess && (unsigned long long)__double_as_longlong(ubd) == key);
                    const uint32_t ness = __popc(__ballot_sync(FULL, ess));
                    if (who == 0u || ness <= 1u) break;
                    const double ub = __longlong_as_double((long long)key);
                    // pass 0 of a two-pass query: a document holding pruned terms of this group and no streamed one is
                    // seen by neither pass (pass 1 drops every document with a group-0 term), so the bound of such a
                    // document includes the other group's terms (ub_oth; 0 in pass 1 and for <= 32 terms)
                    if (!(ub_ne + ub + ub_oth <= (double)BM25X_PRUNE_ALPHA * f.Sk)) break;
                    const int who_i = __ffs(who) - 1;
                    if (C::M <= 8) {
                        ne_list |= (uint32_t)who_i << (4 * n_ne);
                        if (lane == n_ne) ne_prefix_f = __double2float_ru(ub_ne);
                    }
                    n_ne++;
                    ne_mask |= 1u << who_i;
                    ub_ne += ub;
                    changed = true;
                }
                if (changed) {
                    refresh_filter();
                    if (C::ADAPT) {
                        // the pruned terms' rings go back to the budget: the streamed terms get wider windows.  Their rings
                        // move, so what they held beyond rd is fetched again (a few hundred postings, a few times per query)
                        alloc_rings(~ne_mask);
                        uint32_t n = 0;
                        if (lane < (int)m && !((ne_mask >> lane) & 1u)) {
                            wr = rd & ~(C::AL - 1u);
                            n = min(rsize, dfpad - wr);
                        }
                        if (issue_round(n)) {
                            mbar_wait(bar, parity);
                            parity ^= 1u;
                        }
                    }
                }
            }
            const bool act = lane < (int)m && !((ne_mask >> lane) & 1u);
            if constexpr (C::FLAVOUR == RING_SUSPEND) {
                // ---- hand-over: no posting of a streamed run can enter the top-k alone any more (wlim), so the rest of the
                // query only needs doc ids — suspend it for the second phase.  Nothing is in flight here (the round has
                // landed); the pool travels in the query's own output rows, the rest in the record.
                if (!mp && f.tv && __all_sync(FULL, !act || wlim == 0xFFFFFFFFu) &&
                    __reduce_add_sync(FULL, act ? dfj - rd : 0u) >= (uint32_t)BM25X_SUSPEND_MIN) {
                    if (pn > (int)k) pool_cut();
                    const size_t ob = (size_t)qid * k;
                    for (int i = lane; i < pn; i += 32) {
                        p.out_score64[ob + i] = __longlong_as_double((long long)pl.s[i]);
                        p.out_doc[ob + i] = pl.d[i];
                        p.out_score[ob + i] = __uint_as_float(pl.g[i]);
                    }
                    ResumeRec *rec = p.resume + qi;
                    if (lane < 4) {
                        rec->rd[lane] = rd;
                        rec->ne_prefix[lane] = ne_prefix_f;
                    }
                    if (lane == 0) {
                        rec->Sk = f.Sk;
                        rec->ub_ne = ub_ne;
                        rec->lo = lo;
                        rec->pn = (uint32_t)pn;
                        rec->dk = f.dk;
                        rec->tie_sig = f.tie_sig;
                        rec->ne_mask = ne_mask;
                        rec->n_ne = (uint32_t)n_ne;
                        rec->ne_list = ne_list;
                        const uint32_t at = atomicAdd(&p.q2[0], 1u);
                        p.q2[2u + at] = (uint32_t)qi;
                    }
                    suspended = true;
                    break;
                }
            }
            const uint32_t avail_e = min(wr, dfj);
            uint32_t limit = INF;  // runs with postings left in HBM bound the window by their last landed document
            if (act && wr < dfj) limit = ring_doc(myring, (wr - 1u) & rmask);
            uint32_t hi = __reduce_min_sync(FULL, limit);
            bool last = hi == INF;
            uint32_t e = rd;
            {
                // a window usually ends in the last few postings of every ring (all runs advance together): when the posting
                // 32 before the end is still inside the window for every run, 6 search steps over that tail are enough
                const bool tail = act && !last && avail_e - rd > 32u && ring_doc(myring, (avail_e - 33u) & rmask) < hi;
                if (__all_sync(FULL, tail || !act || last)) {
                    if (act) e = last ? avail_e : ring_lower_bound<C, 5>(myring, rmask, avail_e - 32u, avail_e, hi);
                } else if (act) {
                    if (last) e = avail_e;
                    else if (small_rings) e = ring_lower_bound<C, C::LOG_R>(myring, rmask, rd, avail_e, hi);
                    else e = ring_lower_bound<C>(myring, rmask, rd, avail_e, hi);
                }
            }
            // ---- dense or sparse?  (expected number of documents held by two runs in this window) ----
            bool dense = false;
            uint32_t span = 0;
            if (C::M > 1) {
                const uint32_t n = e - rd;
                const uint32_t S = __reduce_add_sync(FULL, n);
                const uint32_t S2 = __reduce_add_sync(FULL, n * n);
                uint32_t hi_eff = hi;
                if (last) hi_eff = __reduce_max_sync(FULL, n ? ring_doc(myring, (e - 1u) & rmask) + 1u : 0u);
                span = hi_eff > lo ? hi_eff - lo : 0u;
                dense = (unsigned long long)S * S - S2 > 2ull * BM25X_RING_DENSE_T * (unsigned long long)span;
                if (dense && span > C::ACC_DOCS) {  // clamp the window to the accumulator: consume the rings partially
                    hi = lo < INF - 1u - C::ACC_DOCS ? lo + C::ACC_DOCS : INF - 1u;
                    last = false;
                    span = C::ACC_DOCS;
                    if (act) e = ring_lower_bound<C>(myring, rmask, rd, e, hi);
                }
            }
            PP_MARK(PP_SETUP);

            uint32_t nc = 0;  // listed candidates (warp-uniform)
            // ---- verification: 32 listed postings at a time ----
            auto verify = [&]() {
                // Three streamed runs (the headline class): TWO lanes per listed posting, each searches one of the two
                // other runs — one search per pass instead of two in a row; the even lane of a pair carries the candidate.
                const bool pairs = C::M == 3 && !C::ADAPT && !dense && m == 3u && ne_mask == 0u;
                // seeded launches with a hit list make room for a pass's candidates BEFORE its searches (a pass of
                // the other lanes then takes at most HCAP candidates)
                constexpr uint32_t GP = C::HITS && C::HCAP < 32 ? (uint32_t)C::HCAP : 32u;
                const uint32_t per_pass = pairs ? 16u : GP;
                PP_COUNT(PP_CANDS, nc);
                for (uint32_t base = 0; base < nc; base += per_pass) {
                    const uint32_t ci = base + (pairs ? (uint32_t)lane >> 1 : (uint32_t)lane);
                    bool has = ci < nc;
                    if constexpr (C::HITS) {
                        has = has && ci < base + per_pass;
                        hit_room(min(per_pass, nc - base));
                    }
                    const uint32_t ent = has ? cand[ci] : 0u;
                    const bool by_doc = (ent >> 15) != 0u;            // dense flavour: document given as offset from lo
                    // seeded launches: run field 31 = a seed (champion of term sidx / SST, slot sidx % SST)
                    const bool is_seed = C::SEEDED && has && !by_doc && ((ent >> 10) & 31u) == 31u;
                    const uint32_t sidx = ent & 0x3FFu;
                    const uint32_t j = by_doc ? 32u : (is_seed ? sidx / C::SST : (ent >> 10) & 31u);
                    Posting own;
                    own.doc = 0;
                    own.w = 0;
                    const uint32_t jbase = C::ADAPT ? __shfl_sync(FULL, rbase, j & 31u) : (j & 31u) * C::R;
                    // doc-id-only rings: the listed posting's word stays in HBM until something needs it — a twin was
                    // found, or run j can still pass alone (wlim): most false alarms of the map never touch HBM
                    const Posting *gown = nullptr;  // DOCRING: &post[posting index] of the listed posting
                    [[maybe_unused]] uint32_t ownix = INF;  // DOCRING: that posting index (relative to pbase)
                    bool solo_j = false;
                    if constexpr (C::DOCRING) {
                        const uint32_t raj = __shfl_sync(FULL, rd, j & 31u);
                        const uint64_t pbj = __shfl_sync(FULL, pbase, j & 31u);
                        solo_j = __shfl_sync(FULL, wlim, j & 31u) != 0xFFFFFFFFu;
                        // seeded launch: a lone streamed holder only matters when a pruned term may hold the document too
                        if constexpr (C::SEEDED) solo_j = false;
                        if constexpr (C::SEEDED) {
                            if (is_seed) own = seeds[sidx];
                        }
                        const uint32_t rmj = C::ADAPT ? __shfl_sync(FULL, rmask, j & 31u) : (uint32_t)C::R - 1u;
                        if (has && !by_doc && !is_seed) {
                            const uint32_t pos = ent & 0x3FFu;
                            own.doc = rings[jbase + pos];
                            ownix = raj + ((pos - raj) & rmj);
                            gown = p.post + pbj + ownix;
                        }
                    } else {
                        if (has && !by_doc) own = rings[jbase + (ent & 0x3FFu)];
                    }
                    const uint32_t doc = by_doc ? lo + (ent & 0x7FFFu) : own.doc;
                    float F = 0.f;
                    uint32_t cnt = 0, sig = SIG_NONE;
                    bool later = false;
                    constexpr bool KEEPW = C::M <= 8;  // posting words of the holders stay in registers for the exact pass
                    uint32_t wv[KEEPW ? C::M : 1];
#pragma unroll
                    for (int i = 0; i < (KEEPW ? C::M : 1); ++i) wv[i] = 0u;
                    // posting word of run i's holder of the document (8-byte rings; the doc-id-only flavours search with
                    // ring_find_pos and never call this)
                    auto holder = [&](int i, uint32_t ib, uint32_t im, uint32_t ai, uint32_t ei) -> uint32_t {
                        if constexpr (C::DOCRING) return 0u;
                        else
                            return (uint32_t)i == j ? own.w
                                                    : (small_rings ? ring_find<C, C::LOG_R>(rings + ib, im, ai, ei, doc)
                                                                   : ring_find<C>(rings + ib, im, ai, ei, doc));
                    };
                    auto filter_term = [&](int i) {
                        const uint32_t ai = __shfl_sync(FULL, rd, i), ei = __shfl_sync(FULL, e, i);
                        const uint32_t ib = ring_base(i), im = ring_mask(i);
                        const float s0 = __shfl_sync(FULL, s0f, i);
                        uint32_t wi = 0u;
                        if (has && !((ne_mask >> i) & 1u)) {
                            wi = holder(i, ib, im, ai, ei);
                            if (wi) {
                                F += score_f32(wi, s0, s1f);
                                cnt++;
                                sig = make_sig(i, wi);
                                later |= (uint32_t)i > j;
                            }
                        }
                        return wi;
                    };
                    if constexpr (C::DOCRING) {
                        // searches first (doc ids in the rings: posting indices of the holders), then the posting words of ALL
                        // holders from HBM with the loads in flight together (one DRAM latency per pass, not one per holder).
                        // A lone posting of a run that cannot pass alone is dropped unread; so is a seed another run holds.
                        if (C::M == 3 && pairs) {
                            const uint32_t o = (lane & 1) ? (j == 2u ? 1u : 2u) : (j == 0u ? 1u : 0u);
                            const uint32_t ao = __shfl_sync(FULL, rd, o), eo = __shfl_sync(FULL, e, o);
                            const uint64_t pbo = __shfl_sync(FULL, pbase, o);
                            uint32_t l = INF;
                            if (has) l = ring_find_pos<C, C::LOG_R>(rings + o * C::R, C::R - 1u, ao, eo, doc);
                            const bool hit = l != INF;
                            const uint32_t hitx = __shfl_xor_sync(FULL, hit ? 1u : 0u, 1);  // (every lane takes part: no short circuit)
                            const bool anyhit = hit || hitx != 0u;
                            const bool live = has && (is_seed ? !anyhit : (anyhit || solo_j));  // (same in both lanes of a pair)
                            PP_MARK(PP_VSEARCH);
                            PP_COUNT(PP_HITS, __popc(__ballot_sync(FULL, live && !(lane & 1))));
                            if constexpr (C::HITS) {
                                // the even lane's row: run j (the listed posting or the seed), run o (its own search),
                                // run ox (the partner's); it waits in the hit list unless a later run holds the document
                                const uint32_t lx = __shfl_xor_sync(FULL, l, 1);
                                const uint32_t ox = (lane & 1) ? (j == 0u ? 1u : 0u) : (j == 2u ? 1u : 2u);
                                const bool later = (l != INF && o > j) || (lx != INF && ox > j);
                                uint32_t hv[C::M];
#pragma unroll
                                for (int i = 0; i < C::M; ++i)
                                    hv[i] = (uint32_t)i == j ? (is_seed ? own.w : ownix)
                                                             : (is_seed ? 0u : ((uint32_t)i == o ? l : ((uint32_t)i == ox ? lx : INF)));
                                hit_append(live && !(lane & 1) && !later, doc, is_seed, hv);
                                PP_MARK(PP_VEXACT);
                                continue;
                            }
                            uint32_t wo = 0u;
                            if (live && hit) wo = __ldg(&(p.post + pbo)[l].w);
                            if (live && !(lane & 1) && !is_seed) own.w = __ldg(&gown->w);
                            const uint32_t wx = __shfl_xor_sync(FULL, wo, 1);  // the partner's run
                            PP_CONSUME(wx, own.w);
                            PP_MARK(PP_VLOAD);
                            const uint32_t ox = (lane & 1) ? (j == 0u ? 1u : 0u) : (j == 2u ? 1u : 2u);
                            has = live && !(lane & 1);
#pragma unroll
                            for (int i = 0; i < C::M; ++i) wv[i] = (uint32_t)i == o ? wo : ((uint32_t)i == ox ? wx : 0u);
                        } else {
                            uint32_t lv[C::M];
                            bool anyhit = false;
#pragma unroll
                            for (int i = 0; i < C::M; ++i) {
                                const uint32_t ai = __shfl_sync(FULL, rd, i), ei = __shfl_sync(FULL, e, i);
                                const uint32_t ib = ring_base(i), im = ring_mask(i);
                                lv[i] = INF;
                                if (i < (int)m && has && (uint32_t)i != j && !((ne_mask >> i) & 1u)) {
                                    lv[i] = small_rings ? ring_find_pos<C, C::LOG_R>(rings + ib, im, ai, ei, doc)
                                                        : ring_find_pos<C>(rings + ib, im, ai, ei, doc);
                                    anyhit = anyhit || lv[i] != INF;
                                }
                            }
                            const bool live = has && (is_seed ? !anyhit : (by_doc || anyhit || solo_j));
                            PP_MARK(PP_VSEARCH);
                            PP_COUNT(PP_HITS, __popc(__ballot_sync(FULL, live)));
                            if constexpr (C::HITS) {
                                // a live row waits in the hit list unless a later run holds the document; a streamed
                                // (or dense-window) document needs a second holder: one holder alone is a seed's business
                                bool later = false;
                                uint32_t nh = by_doc ? 0u : 1u, hv[C::M];
#pragma unroll
                                for (int i = 0; i < C::M; ++i) {
                                    later |= lv[i] != INF && (uint32_t)i > j;
                                    nh += lv[i] != INF ? 1u : 0u;
                                    hv[i] = (uint32_t)i == j ? (is_seed ? own.w : ownix) : (is_seed ? 0u : lv[i]);
                                }
                                hit_append(live && !later && (is_seed || nh >= 2u), doc, is_seed, hv);
                                PP_MARK(PP_VEXACT);
                                continue;
                            }
#pragma unroll
                            for (int i = 0; i < C::M; ++i) {
                                const uint64_t pbi = __shfl_sync(FULL, pbase, i);
                                if (live && lv[i] != INF) wv[i] = __ldg(&(p.post + pbi)[lv[i]].w);
                            }
                            if (live && !by_doc && !is_seed) own.w = __ldg(&gown->w);
#pragma unroll
                            for (int i = 0; i < C::M; ++i) PP_CONSUME(wv[i], own.w);
                            PP_MARK(PP_VLOAD);
                            has = live;
                        }
#pragma unroll
                        for (int i = 0; i < C::M; ++i) {
                            const float s0 = __shfl_sync(FULL, s0f, i);
                            const uint32_t wi = (uint32_t)i == j ? own.w : wv[i];
                            if (has && wi) {
                                F += score_f32(wi, s0, s1f);
                                cnt++;
                                sig = make_sig(i, wi);
                                later |= (uint32_t)i > j;
                            }
                            wv[i] = has ? wi : 0u;
                        }
                        // seeded launch: single-term documents are in the pool already (or lost to better ones)
                        // (a seed that another term holds is the stream's business; a streamed posting that no other term
                        // holds is a seed's)
                        if constexpr (C::SEEDED) has = has && (is_seed ? cnt == 1u : !(ne_mask == 0u && cnt == 1u));
                    } else if (C::M == 3 && pairs) {
                        if constexpr (C::M == 3) {
                            // my run to search: the first (even lane) or second (odd lane) of the two runs other than j
                            const uint32_t o = (lane & 1) ? (j == 2u ? 1u : 2u) : (j == 0u ? 1u : 0u);
                            const uint32_t ao = __shfl_sync(FULL, rd, o), eo = __shfl_sync(FULL, e, o);
                            uint32_t wo = 0u;
                            if (has) wo = ring_find<C, C::LOG_R>(rings + o * C::R, C::R - 1u, ao, eo, doc);
                            const uint32_t wx = __shfl_xor_sync(FULL, wo, 1);  // the partner's run
                            const uint32_t ox = (lane & 1) ? (j == 0u ? 1u : 0u) : (j == 2u ? 1u : 2u);
                            has = has && !(lane & 1);
#pragma unroll
                            for (int i = 0; i < 3; ++i) {
                                const float s0 = __shfl_sync(FULL, s0f, i);
                                const uint32_t wi = (uint32_t)i == j ? own.w : ((uint32_t)i == o ? wo : ((uint32_t)i == ox ? wx : 0u));
                                if (has && wi) {
                                    F += score_f32(wi, s0, s1f);
                                    cnt++;
                                    sig = make_sig(i, wi);
                                    later |= (uint32_t)i > j;
                                }
                                wv[i] = has ? wi : 0u;
                            }
                        }
                    } else if constexpr (KEEPW) {
#pragma unroll
                        for (int i = 0; i < C::M; ++i)
                            if (i < (int)m) wv[i] = filter_term(i);
                    } else {
#pragma unroll 1
                        for (int i = 0; i < (int)m; ++i) filter_term(i);
                    }
                    // the last streamed run holding the document emits it: its posting always detects the others
                    bool keep = has && !later && wfilter_pass(f, F, cnt == 1 ? sig : SIG_NONE, doc);
                    if (keep && p.allow && !((p.allow[doc >> 3] >> (doc & 7u)) & 1u)) keep = false;
                    if (__any_sync(FULL, keep)) {
                        // exact re-score in the reference's operation order; pruned terms are probed in HBM
                        double Sx = 0.0;
                        uint32_t cnt_all = 0;
                        auto exact_term = [&](int i, uint32_t wi) {
                            const double s0 = __shfl_sync(FULL, s0d, i);
                            if ((ne_mask >> i) & 1u) {
                                const uint64_t pb = __shfl_sync(FULL, pbase, i), bb = __shfl_sync(FULL, bbase, i);
                                const uint32_t nbq = __shfl_sync(FULL, nbj, i), dfq = __shfl_sync(FULL, dfj, i);
                                wi = 0u;
                                if (keep) {
                                    const uint32_t l = probe_block(p, bb, nbq, doc, probe_steps);
                                    if (l > 0u) wi = probe_in_block(p, pb, dfq, l - 1u, doc, probe_steps);
                                    if (wi) sig = make_sig(i, wi);
                                }
                            }
                            if (keep && wi) {
                                Sx = __dadd_rn(Sx, score_f64(wi, s0, p.s1d));
                                cnt_all++;
                            }
                        };
                        if constexpr (KEEPW) {
                            if (ne_mask) {
                                // pruned terms: probe in HBM, largest bound first; Fres = f32 score over the holders
                                // found so far, rest = Σ bounds of the pruned terms not probed yet
                                float Fres = F;
                                for (int t = n_ne - 1; t >= 0; --t) {
                                    const int i = (int)((ne_list >> (4 * t)) & 15u);
                                    const uint64_t pb = __shfl_sync(FULL, pbase, i), bb = __shfl_sync(FULL, bbase, i);
                                    const uint32_t nbq = __shfl_sync(FULL, nbj, i), dfq = __shfl_sync(FULL, dfj, i);
                                    const float s0 = __shfl_sync(FULL, s0f, i);
                                    const float rest = __shfl_sync(FULL, ne_prefix_f, t);
                                    uint32_t wi = 0u;
                                    if (keep) {
                                        const uint32_t l = probe_block(p, bb, nbq, doc, probe_steps);
                                        bool inside = false;
                                        if (l > 0u && __ldg(&p.blk[bb + l - 1u].y) >= doc) {
                                            // block-max test before the deep seek (search.rs:193-203)
                                            if (Fres + __ldg(&p.blk_ub[bb + l - 1u]) + rest < FloT) keep = false;
                                            else inside = true;
                                        }
                                        if (inside) wi = probe_in_block(p, pb, dfq, l - 1u, doc, probe_steps);
                                        if (wi) {
                                            Fres += score_f32(wi, s0, s1f);
                                            sig = make_sig(i, wi);
                                        }
                                        if (keep && Fres + rest < FloT) keep = false;
                                    }
#pragma unroll
                                    for (int ii = 0; ii < C::M; ++ii)
                                        if (ii == i) wv[ii] = wi;
                                }
                            }
                            if (__any_sync(FULL, keep)) Sx = exact_sum(keep, wv, cnt_all);
                        } else {
                            // posting word of `doc` in a term that is no lane of this pass (two-pass queries)
                            auto probe_term = [&](uint32_t term) -> uint32_t {
                                const uint32_t dft = p.df[term];
                                const uint32_t l = probe_block(p, p.blk_off[term], (dft + BM25X_BLOCK - 1) / BM25X_BLOCK, doc, probe_steps);
                                return l > 0u ? probe_in_block(p, p.post_off[term], dft, l - 1u, doc, probe_steps) : 0u;
                            };
                            if (mp && pass == 1) {  // documents holding a first-group term were emitted by the first pass
                                for (uint32_t u = 0; u < on && __any_sync(FULL, keep); ++u) {
                                    const uint32_t term = p.q_terms[obase + u];
                                    if (keep && probe_term(term)) keep = false;
                                }
                            }
                            // both groups merged in ascending term id: the reference order of the f64 sum
                            uint32_t ia = 0, iob = 0;
#pragma unroll 1
                            while (ia < m || iob < on) {
                                const uint32_t ta = ia < m ? p.q_terms[t0 + ia] : INF, tb = iob < on ? p.q_terms[obase + iob] : INF;
                                if (ta < tb) {
                                    const int i = (int)ia;
                                    const uint32_t ai = __shfl_sync(FULL, rd, i), ei = __shfl_sync(FULL, e, i);
                                    const uint32_t ib = ring_base(i), im = ring_mask(i);
                                    uint32_t wi = 0u;
                                    if (keep && !((ne_mask >> i) & 1u)) wi = holder(i, ib, im, ai, ei);
                                    exact_term(i, wi);
                                    ia++;
                                } else {
                                    if (pass == 0) {  // first pass: the second group's terms are probed for the survivors
                                        const double s0 = p.s0d[tb];
                                        uint32_t wi = 0u;
                                        if (keep) wi = probe_term(tb);
                                        if (keep && wi) {
                                            Sx = __dadd_rn(Sx, score_f64(wi, s0, p.s1d));
                                            cnt_all++;
                                        }
                                    }
                                    iob++;
                                }
                            }
                        }
                        if constexpr (C::SEEDED) keep = keep && (is_seed ? cnt_all == 1u : cnt_all != 1u);  // (pruned terms probed)
                        pool_insert(keep, Sx, doc, cnt_all == 1 ? sig : SIG_NONE);
                    }
                    PP_MARK(PP_VEXACT);
                }
                __syncwarp();  // every lane has read its entries before the producers refill the list
                nc = 0;
            };

            // ---- candidate production (resumable) + ONE verification site ----
            // sparse window: runs in ascending order; each run tests its documents against the marks of the earlier runs,
            // then marks them.  dense window: scores summed in an f32 accumulator indexed by doc - lo (in the map's
            // memory; docs are distinct inside a run: plain read-modify-write, __syncwarp between runs), then scanned.
            uint32_t todo = 0u, ra = 0u, ree = 0u, wl = 0u, tw = 0u, tdk = 0u, pb = 0u, dbase = 0u, rm = 1u;
            int rj = -1, variant = 0;
            uint32_t ss = 0u;  // seeded launches: next slice (term, 32 slots) of the seed table to look at in this window
            bool multi = false;
            const uint4 *rg = nullptr;
            const uint4 *gq = nullptr;  // DOCRING: the current run's 8-byte postings in HBM (single-term test only)
            int myvariant = 0;  // lane j: loop variant of run j in this window (4: single-term test, 2: test, 1: mark)
            if (!dense) {
                todo = __ballot_sync(FULL, act && e > rd);
                multi = C::M > 1 && __popc(todo) > 1;
                if (multi) {  // clear the map for this window
                    for (int i = lane; i < (int)(C::MAP_BYTES / 16u); i += 32) ((uint4 *)map)[i] = make_uint4(0, 0, 0, 0);
                    __syncwarp();
                }
                PP_MARK(PP_CLEAR);
                // wlim == ~0: no single-term posting of the run can pass → the loop variant without that test; the first
                // non-empty run has nothing to test against, the last one nobody to mark for
                myvariant = (!C::SEEDED && wlim != 0xFFFFFFFFu ? 4 : 0) | (multi && lane != __ffs(todo) - 1 ? 2 : 0) |
                            (multi && lane != 31 - __clz(todo) ? 1 : 0);
            } else {
                float *acc = (float *)map;
                for (uint32_t i = lane; i < (span + 3u) / 4u; i += 32) ((float4 *)acc)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                __syncwarp();
                uint32_t td = __ballot_sync(FULL, act && e > rd);
                while (td) {
                    const int j = __ffs(td) - 1;
                    td &= td - 1u;
                    const uint32_t a = __shfl_sync(FULL, rd, j), ee = __shfl_sync(FULL, e, j);
                    const float s0 = __shfl_sync(FULL, s0f, j);
                    const RT *rgp = rings + ring_base(j);
                    const uint32_t jm = ring_mask(j);
                    if constexpr (C::DOCRING) {  // the posting words of a dense window come straight from HBM
                        const Posting *gp = p.post + __shfl_sync(FULL, pbase, j);
                        for (uint32_t i = a + lane; i < ee; i += 32) acc[rgp[i & jm] - lo] += score_f32(__ldg(&gp[i].w), s0, s1f);
                    } else {
                        for (uint32_t i = a + lane; i < ee; i += 32) {
                            const Posting v = rgp[i & jm];
                            acc[v.doc - lo] += score_f32(v.w, s0, s1f);
                        }
                    }
                    __syncwarp();
                }
            }
            // Up to TMAX trips of TRIP postings of the current run, then ONE compaction of the detected postings (a bit
            // per posting slot in `hm`: per-trip ballot compaction cost as much as the test itself).
            auto run = [&](auto test_c, auto mark_c, auto solo_c) {
                constexpr bool TEST = decltype(test_c)::value, MARK = decltype(mark_c)::value;
                constexpr bool SOLO = decltype(solo_c)::value;
                const uint32_t pb0 = pb;
                uint32_t hm = 0u;
#pragma unroll 1
                for (int t = 0; t < C::TMAX && pb < ree; ++t, pb += C::TRIP) {
                    uint4 q[C::U];
                    uint32_t ix[C::U];
                    // DOCRING: tf / fieldnorm words only while a posting of this run can still pass alone (loop variants
                    // with the single-term test): two 16-byte loads per four doc ids, straight from HBM / L2
                    uint4 gw[C::DOCRING && SOLO ? C::U : 1][2];
#pragma unroll
                    for (int u = 0; u < C::U; ++u) {
                        ix[u] = pb + (uint32_t)C::E * (uint32_t)(lane + 32 * u);
                        q[u] = rg[(ix[u] / (uint32_t)C::E) & (rm / (uint32_t)C::E)];
                        if constexpr (C::DOCRING && SOLO) {
                            gw[u][0] = gw[u][1] = make_uint4(0u, 0u, 0u, 0u);
                            if (ix[u] < ree) {  // ix is a multiple of 4 and the lists are padded to 4: in bounds
                                gw[u][0] = __ldg(gq + (ix[u] >> 1));
                                gw[u][1] = __ldg(gq + (ix[u] >> 1) + 1);
                            }
                        }
                    }
                    uint32_t bits = 0u;
                    auto body = [&](auto check_c) {
                        // trips at the ends of the range: which of the lane's posting slots lie in [ra, ree), once per lane
                        // and trip; the others neither mark nor test (a mark from outside the window would add false
                        // alarms, a hit there would list a posting of another window)
                        constexpr bool CHECK = decltype(check_c)::value;
                        uint32_t vm = 0xFFFFFFFFu;
                        if constexpr (CHECK) {
                            vm = 0u;
#pragma unroll
                            for (int u = 0; u < C::U; ++u) {
                                // slots below ra: at most E - 1 (a run's first trip starts at ra & ~(E - 1)); slots from
                                // ree on: any number
                                constexpr uint32_t ALL = (1u << C::E) - 1u;
                                const int below = max((int)(ra - ix[u]), 0), beyond = max((int)(ix[u] + C::E - ree), 0);
                                vm |= ((ALL << below) & (ALL >> min(beyond, C::E))) << (C::E * u);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < C::U; ++u) {
#pragma unroll
                            for (int h = 0; h < C::E; ++h) {
                                uint32_t doc, w = 0u;
                                if constexpr (C::DOCRING) {
                                    doc = h == 0 ? q[u].x : (h == 1 ? q[u].y : (h == 2 ? q[u].z : q[u].w));
                                    if constexpr (SOLO) w = (h & 1) ? gw[u][h >> 1].w : gw[u][h >> 1].y;
                                } else {
                                    doc = h ? q[u].z : q[u].x;
                                    w = h ? q[u].w : q[u].y;
                                }
                                const bool valid = (vm >> (C::E * u + h)) & 1u;
                                bool c = false;
                                if (TEST || MARK) {
                                    uint32_t msk;
                                    uint32_t *cell = (uint32_t *)map + map_word<C>(doc, msk);
                                    // an invalid slot ORs nothing in (an atomic with an empty mask: no branch around it)
                                    // and its test is masked off below; the word is in the map whatever the slot holds
                                    const uint32_t mark = CHECK && !valid ? 0u : msk;
                                    uint32_t old = 0u;
                                    if (TEST && MARK) {
                                        // one atomic tests and marks: the old word also holds this run's earlier marks,
                                        // which can only add false alarms (the verification drops them), never hide a
                                        // mark of an earlier run
                                        old = atomicOr(cell, mark);
                                    } else {
                                        if (TEST) old = *cell;
                                        if (MARK) atomicOr(cell, mark);
                                    }
                                    // hit: every bit of msk was set already (one LOP3 sets the predicate, one predicated
                                    // add records it)
                                    if (TEST) c = (msk & ~old) == 0u;
                                }
                                if (SOLO) c = c | ((w > wl) & !((w == tw) & (doc > tdk)));  // bitwise: no branches
                                if (c) bits += 1u << (C::E * u + h);
                            }
                        }
                        if constexpr (CHECK) bits &= vm;
                    };
                    if (pb >= ra && pb + C::TRIP <= ree) body(std::false_type());
                    else body(std::true_type());
                    hm |= bits << (C::PL * t);
                }
                PP_MARK(PP_STREAM);
                // compaction: one listed posting per lane and round.  Bit b = PL·t + E·u + h of hm is posting
                // pb0 + t·TRIP + E·(lane + 32·u) + h = pb0 + E·lane + 32·(b & ~(E - 1)) + (b & (E - 1)).
                const uint32_t lane0 = pb0 + (uint32_t)C::E * (uint32_t)lane, rtag = (uint32_t)rj << 10;
                for (;;) {
                    const uint32_t bal = __ballot_sync(FULL, hm != 0u);
                    if (!bal) break;
                    if (hm) {
                        const uint32_t b = (uint32_t)__ffs(hm) - 1u;
                        hm &= hm - 1u;
                        const uint32_t idx = lane0 + b + 31u * (b & ~((uint32_t)C::E - 1u));
                        cand[nc + __popc(bal & lt_mask)] = (uint16_t)((idx & rm) | rtag);
                    }
                    nc += __popc(bal);
                }
                PP_MARK(PP_COMPACT);
            };
            // Producer loop: runs (or the accumulator scan) list candidates until the list wants to be verified or the
            // window is done; ONE verification site after it.
            bool more = true;
            while (more) {
                bool seeds_pending = false;
                if constexpr (C::SEEDED) {
                    // the seeds of this doc window join the candidate list first (entry: run field 31 | seed slot); the
                    // rings hold every run's postings of the window, so the ONE verification site below tells whether
                    // another term holds the document
                    const uint32_t slices = (min(k, (uint32_t)BM25X_CHAMP_L) + 31u) >> 5;  // per term
#pragma unroll 1
                    while (ss < (uint32_t)C::M * slices && nc <= 64u) {
                        uint32_t jj = ss, r = (uint32_t)lane;
                        if constexpr (C::SST > 32u) {
                            jj = ss / slices;
                            r += (ss % slices) * 32u;
                        }
                        ++ss;
                        if (jj >= m || ((ne_mask >> jj) & 1u)) continue;  // a pruned term's documents cannot enter
                        const uint32_t d = seeds[jj * C::SST + r].doc;
                        const bool inw = d >= lo && d < hi;
                        const uint32_t bal = __ballot_sync(FULL, inw);
                        if (inw) cand[nc + __popc(bal & lt_mask)] = (uint16_t)((31u << 10) | (jj * C::SST + r));
                        nc += __popc(bal);
                    }
                    seeds_pending = ss < (uint32_t)C::M * slices;
                    PP_MARK(PP_SEEDS);
                }
                if (seeds_pending) {
                    __syncwarp();  // list full: verify, then go on with the seeds
                } else if (!dense) {
                    for (;;) {
                        if (pb >= ree) {  // next run
                            if (rj >= 0) __syncwarp();  // this run's marks are visible to the next run's tests
                            if (!todo) {
                                more = false;
                                break;
                            }
                            rj = __ffs(todo) - 1;
                            todo &= todo - 1u;
                            ra = __shfl_sync(FULL, rd, rj);
                            ree = __shfl_sync(FULL, e, rj);
                            wl = __shfl_sync(FULL, wlim, rj);
                            tw = __shfl_sync(FULL, tiew, rj);
                            variant = __shfl_sync(FULL, myvariant, rj);
                            rg = (const uint4 *)(rings + ring_base(rj));
                            if constexpr (C::DOCRING) gq = (const uint4 *)(p.post + __shfl_sync(FULL, pbase, rj));
                            rm = ring_mask(rj);
                            tdk = f.tie_dk;  // snapshot with tw: a stale (looser) pair stays valid, thresholds only tighten
                            pb = ra & ~((uint32_t)C::E - 1u);
                        }
                        if constexpr (C::SEEDED) {  // no loop variant with the single-term test
                            switch (variant & 3) {
                                case 0: pb = ree; break;  // nothing to learn from this run in this window
                                case 3: run(std::true_type(), std::true_type(), std::false_type()); break;
                                case 1: run(std::false_type(), std::true_type(), std::false_type()); break;
                                default: run(std::true_type(), std::false_type(), std::false_type()); break;
                            }
                        } else {
                            switch (variant) {
                                case 0: pb = ree; break;  // nothing to learn from this run in this window
                                case 3: run(std::true_type(), std::true_type(), std::false_type()); break;
                                case 1: run(std::false_type(), std::true_type(), std::false_type()); break;
                                case 2: run(std::true_type(), std::false_type(), std::false_type()); break;
                                case 4: run(std::false_type(), std::false_type(), std::true_type()); break;
                                case 5: run(std::false_type(), std::true_type(), std::true_type()); break;
                                case 6: run(std::true_type(), std::false_type(), std::true_type()); break;
                                default: run(std::true_type(), std::true_type(), std::true_type()); break;
                            }
                        }
                        if (nc > 64u) break;
                    }
                    __syncwarp();  // the listed entries are visible to every lane
                } else {
                    const float *acc = (const float *)map;
                    while (dbase < span && nc <= 64u) {
                        const uint32_t o = dbase + lane;
                        const float F = o < span ? acc[o] : 0.f;
                        const bool c = F > 0.f && F >= f.Flo;
                        const uint32_t mc = __ballot_sync(FULL, c);
                        if (c) cand[nc + __popc(mc & lt_mask)] = (uint16_t)(0x8000u | o);
                        nc += __popc(mc);
                        dbase += 32;
                    }
                    __syncwarp();
                    more = dbase < span;
                }
                if (nc) verify();
            }
            rd = e;
            lo = hi;
            if (last) break;
            // ---- refill: everything this chunk freed (the ring is one window, refilled after it: the load is exposed,
            // but the bytes should already sit in L2 — half the ring memory per posting in flight, i.e. more resident warps)
            uint32_t n = 0;
            if (act && wr < dfpad) {
                n = min((rsize - (wr - rd)) & ~(C::AL - 1u), dfpad - wr);
                if (n < rsize / 4 && wr - rd >= rsize / 4) n = 0;  // no small top-ups
            }
            inflight = issue_round(n);
            if (n > 0 && wr < dfpad) {  // the round after this one: into L2 while this chunk's successor is processed
                const uint32_t pn_ = min(rsize, dfpad - wr);
                if constexpr (C::DOCRING) {
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.pdoc + pbase + wr), "r"(pn_ * 4u) : "memory");
                    // while postings of this run can still pass alone, the loop also reads their tf / fieldnorm words
                    if (wlim != 0xFFFFFFFFu)
                        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.post + pbase + wr), "r"(pn_ * 8u) : "memory");
                } else {
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.post + pbase + wr), "r"(pn_ * 8u) : "memory");
                }
            }
            PP_MARK(PP_END);
        }
        if constexpr (C::HITS) hit_drain();
        // ---- Results::into_sorted_vec (search.rs:281) (after the last pass; between passes: a tidy pool and threshold) ----
        if (pn > 0 && !suspended) pool_cut();
        }  // passes
        if (suspended) {  // no result rows yet; the statistics of this phase are final
            if (p.fetched) {
                fetched += probe_steps;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) fetched += __shfl_xor_sync(FULL, fetched, o);
                if (lane == 0) atomicAdd(p.fetched, fetched);
            }
            __syncwarp();
            continue;
        }
        const size_t obase = (size_t)qid * k;
        for (uint32_t i = lane; i < k; i += 32) {
            uint32_t d = INF;
            double sc = 0.0;
            if ((int)i < pn) {
                d = pl.d[i];
                sc = __longlong_as_double((long long)pl.s[i]);
            }
            p.out_doc[obase + i] = d;
            p.out_score[obase + i] = (float)sc;
            if (p.out_score64) p.out_score64[obase + i] = sc;
            if (p.out_payload) {
                uint16_t a = 0, b = 0, cc = 0;
                if ((int)i < pn) {
                    a = p.payload[(size_t)d * 3 + 0];
                    b = p.payload[(size_t)d * 3 + 1];
                    cc = p.payload[(size_t)d * 3 + 2];
                }
                p.out_payload[(obase + i) * 3 + 0] = a;
                p.out_payload[(obase + i) * 3 + 1] = b;
                p.out_payload[(obase + i) * 3 + 2] = cc;
            }
        }
        if (lane == 0) p.out_n[qid] = (uint32_t)pn;
        if (p.fetched) {
            unsigned long long fsum = (unsigned long long)fetched + probe_steps;  // + block-table entries / postings read by the probes of pruned terms
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) fsum += __shfl_xor_sync(FULL, fsum, o);
            if (lane == 0) atomicAdd(p.fetched, fsum);
        }
#ifdef BM25X_PHASE_PROF
        PP_MARK(PP_QUERY);
        if constexpr (C::SEEDED) {
            if (lane < PP_SLOTS) atomicAdd(&g_phase_prof[lane], (unsigned long long)pp_acc);
            pp_acc = 0u;
        }
#endif
        __syncwarp();
    }
}

}  // namespace
