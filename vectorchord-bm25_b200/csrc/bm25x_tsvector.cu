// bm25x_tsvector.cu — the tsvector casts on the GPU (DESIGN §4.10): documents and queries taken as PostgreSQL tsvectors,
// as every way into the reference takes them.
//
// cast_tsvector_to_document / cast_tsvector_to_query (src/datatype/tsvector.rs:84-105) intern every lexeme of a vector
// (vector::intern, crates/bm25/src/vector.rs:19-35), sort by key and merge equal keys (document: the position counts
// summed with saturation, tsvector.rs:107-127).  Here, over chunks of whole vectors:
//   1. k_tsv_intern: one thread per WordEntry.  The lexeme is copied (short) or hashed (BLAKE3 keyed_hash in registers,
//      at most 2 chunks + 1 parent), and the key goes out as Key128 tagged with its vector;
//   2. a CUB radix sort by (vector, key) and a reduce by key with a saturating add merge the runs;
//   3. k_tsv_emit writes each merged element at its place in the device-resident output (raw key bytes and tf, or the
//      key's ordinal in an index's vocabulary), counts it into its vector's row and sums its vector's length.
// Row offsets come from the row counts by a host scan once every chunk has run, so that a refused cast writes nothing.
// The build from tsvectors hands the device-resident keyed CSR to the build from documents (documents_build): the keys
// never travel to the host.  The sharded build casts each shard's slice on its device and hands only its distinct keys
// and their counts to the host, which merges them into the vocabulary; each shard's keys then become ordinals in place
// and the build from documents inverts them without keys.  A growing segment's insert (tsvector_rows) numbers the keys its sealed vocabulary lacks:
// k_tsv_missing compacts them, a radix sort and a unique give the call's distinct ones ascending, the host numbers
// those, k_tsv_fresh hands each element its ordinal and a segmented sort puts every row back in ordinal order.
#include <string.h>

#include <algorithm>
#include <queue>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cub/device/device_select.cuh>

#include "bm25x_build.h"
#include "bm25x_keys.cuh"

namespace {

constexpr uint64_t CHUNK_ENT = 1ull << 22;    // entries per upload chunk
constexpr uint64_t CHUNK_BYTES = 1ull << 26;  // lexeme-area bytes per upload chunk
constexpr uint64_t CHUNK_VEC = 1ull << 22;    // vectors per upload chunk (empty vectors cost no entry)

// ---- BLAKE3 keyed_hash, the first 16 bytes, of one lexeme of at most 2047 bytes (WordEntry.len has 11 bits) ----

struct Seed {  // the 32-byte key as eight little-endian words, passed by value (kernel parameter space)
    uint32_t w[8];
};
enum : uint32_t { CHUNK_START = 1, CHUNK_END = 2, PARENT = 4, ROOT = 8, KEYED_HASH = 16 };
constexpr uint32_t IV0 = 0x6A09E667u, IV1 = 0xBB67AE85u, IV2 = 0x3C6EF372u, IV3 = 0xA54FF53Au;

__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ void g(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &d, uint32_t mx, uint32_t my) {
    a = a + b + mx;
    d = rotr(d ^ a, 16);
    c = c + d;
    b = rotr(b ^ c, 12);
    a = a + b + my;
    d = rotr(d ^ a, 8);
    c = c + d;
    b = rotr(b ^ c, 7);
}

// The compression function: cv = the first 8 words of its output.  Every index is a constant once the rounds are
// unrolled, so the state and the message stay in registers; the message permutation is register renaming.
__device__ __forceinline__ void compress(uint32_t cv[8], const uint32_t block[16], uint32_t counter, uint32_t block_len,
                                         uint32_t flags) {
    uint32_t s[16] = {cv[0], cv[1], cv[2], cv[3], cv[4], cv[5], cv[6], cv[7], IV0, IV1, IV2, IV3, counter, 0u,
                      block_len, flags};
    uint32_t m[16];
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = block[i];
#pragma unroll
    for (int r = 0; r < 7; r++) {
        g(s[0], s[4], s[8], s[12], m[0], m[1]);
        g(s[1], s[5], s[9], s[13], m[2], m[3]);
        g(s[2], s[6], s[10], s[14], m[4], m[5]);
        g(s[3], s[7], s[11], s[15], m[6], m[7]);
        g(s[0], s[5], s[10], s[15], m[8], m[9]);
        g(s[1], s[6], s[11], s[12], m[10], m[11]);
        g(s[2], s[7], s[8], s[13], m[12], m[13]);
        g(s[3], s[4], s[9], s[14], m[14], m[15]);
        const uint32_t t[16] = {m[2], m[6], m[3], m[10], m[7], m[0], m[4], m[13],
                                m[1], m[11], m[12], m[5], m[9], m[14], m[15], m[8]};  // MSG_PERMUTATION
#pragma unroll
        for (int i = 0; i < 16; i++) m[i] = t[i];
    }
#pragma unroll
    for (int i = 0; i < 8; i++) cv[i] = s[i] ^ s[i + 8];
}

// Block b of the message p[0..len): 64 bytes from offset 64 b, zero past len, as sixteen little-endian words.
__device__ __forceinline__ void load_block(const uint8_t *__restrict__ p, uint32_t len, uint32_t b, uint32_t m[16]) {
    const uint32_t off = 64 * b;
#pragma unroll
    for (int w = 0; w < 16; w++) {
        uint32_t v = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t at = off + 4 * w + j;
            if (at < len) v |= (uint32_t)p[at] << (8 * j);
        }
        m[w] = v;
    }
}

// The first four words of blake3::keyed_hash(seed, p[0..len)), len <= 2047: one chunk is the root; two chunks (1024
// bytes, then the rest) are joined by a parent, which is the root.
__device__ __forceinline__ void blake3_keyed16(const Seed &seed, const uint8_t *__restrict__ p, uint32_t len,
                                               uint32_t out[4]) {
    uint32_t cv[8], cv0[8], m[16];
#pragma unroll
    for (int i = 0; i < 8; i++) cv[i] = seed.w[i];
    const bool two = len > 1024;
    const uint32_t nb = len == 0 ? 1u : (len + 63) / 64;  // blocks over both chunks (chunk 0 holds 16 when two)
    for (uint32_t b = 0; b < nb; b++) {
        const uint32_t chunk = b >= 16 ? 1u : 0u, first = b - 16 * chunk;
        if (b == 16) {
#pragma unroll
            for (int i = 0; i < 8; i++) {
                cv0[i] = cv[i];
                cv[i] = seed.w[i];
            }
        }
        load_block(p, len, b, m);
        const bool last = b + 1 == nb, chunk_last = last || (two && b == 15);
        const uint32_t flags = KEYED_HASH | (first == 0 ? CHUNK_START : 0u) | (chunk_last ? CHUNK_END : 0u) |
                               (last && !two ? ROOT : 0u);
        compress(cv, m, chunk, min(64u, len - 64 * b), flags);
    }
    if (two) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            m[i] = cv0[i];
            m[i + 8] = cv[i];
            cv[i] = seed.w[i];
        }
        compress(cv, m, 0, 64, KEYED_HASH | PARENT | ROOT);
    }
#pragma unroll
    for (int i = 0; i < 4; i++) out[i] = cv[i];
}

// ---- the cast ----

// A key tagged with the vector that holds it (the vector local to its chunk): sorted by (vec, hi, lo).
struct VKey {
    uint64_t hi, lo;
    uint32_t vec;
};
struct VKeyBits {  // CUB's radix decomposer, most significant first
    __host__ __device__ ::cuda::std::tuple<uint32_t &, uint64_t &, uint64_t &> operator()(VKey &k) const {
        return {k.vec, k.hi, k.lo};
    }
};
__host__ __device__ __forceinline__ bool operator==(const VKey &a, const VKey &b) {  // the merge's run test
    return a.vec == b.vec && a.hi == b.hi && a.lo == b.lo;
}
struct SatAdd {  // Saturating<u32> sum (tsvector.rs:115-120)
    __host__ __device__ uint32_t operator()(uint32_t a, uint32_t b) const {
        const uint32_t s = a + b;
        return s < a ? 0xFFFFFFFFu : s;
    }
};

// One thread per entry of a chunk of nv vectors: entries of vector u are [eoff[u], eoff[u+1]) (rebased to the chunk),
// its area bytes + boff[u] (rebased).  key[i] = the interned lexeme (vector::intern) tagged with u; cnt[i] = its
// position count (document mode; the host checked that every entry has one).
__global__ void k_tsv_intern(const uint32_t *__restrict__ ent, uint64_t n, const uint64_t *__restrict__ eoff,
                             const uint64_t *__restrict__ boff, uint32_t nv, const uint8_t *__restrict__ bytes,
                             const Seed seed, int as_query, VKey *__restrict__ key, uint32_t *__restrict__ cnt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t u = owner_of(eoff, nv, i), e = ent[i];
    const uint32_t len = (e >> 1) & 0x7FFu, pos = e >> 12;
    const uint8_t *__restrict__ area = bytes + boff[u];
    const uint8_t *__restrict__ lex = area + pos;
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    bool nul = false;
    if (len < 16) {
#pragma unroll
        for (uint32_t j = 0; j < 15; j++)
            if (j < len) {
                const uint32_t c = lex[j];
                nul |= c == 0;
                w[j >> 2] |= c << (8 * (j & 3));
            }
    }
    if (len >= 16 || nul) {
        blake3_keyed16(seed, lex, len, w);
        if ((w[3] >> 24) == 0) w[3] |= 1u << 24;  // vector.rs:30-32: a hashed key never ends in a zero byte
    }
    VKey k;
    k.hi = bswap64((uint64_t)w[0] | (uint64_t)w[1] << 32);
    k.lo = bswap64((uint64_t)w[2] | (uint64_t)w[3] << 32);
    k.vec = u;
    key[i] = k;
    if (!as_query) {
        const uint32_t at = (pos + len + 1) & ~1u;  // SHORTALIGN(pos + len): the u16 count of the positions
        cnt[i] = (uint32_t)area[at] | (uint32_t)area[at + 1] << 8;
    }
}

// One thread per merged element i < *runs of a chunk whose vectors start at global vector v0 and whose elements go to
// global element base + i: raw key bytes and tf (when given), or the ordinal of the key in the sorted vocabulary
// (BM25X_TERM_MISSING when absent, address_tokens::read).  rows[v] counts the elements of vector v; document mode also
// len[v] += tf, and the first vector with a merged tf of 0 / of 2^24 or more into flags[0] / flags[1].
__global__ void k_tsv_emit(const VKey *__restrict__ key, const uint32_t *__restrict__ tf, const int64_t *__restrict__ runs,
                           uint32_t v0, uint64_t base, int as_query, ulonglong2 *__restrict__ out_key,
                           uint32_t *__restrict__ out_tf, const Key128 *__restrict__ vocab, uint32_t T,
                           uint32_t *__restrict__ out_ord, uint32_t *__restrict__ rows, uint64_t *__restrict__ len,
                           uint32_t *__restrict__ flags) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < (uint64_t)*runs;
    const VKey k = live ? key[i] : VKey{0, 0, 0xFFFFFFFFu};
    const uint32_t v = v0 + k.vec;
    const uint32_t same = __match_any_sync(0xFFFFFFFFu, k.vec);
    if (!live) return;
    if ((threadIdx.x & 31) == (unsigned)(__ffs(same) - 1)) atomicAdd(&rows[v], (uint32_t)__popc(same));
    const Key128 kk{k.hi, k.lo};
    if (out_key) out_key[base + i] = raw_of(kk);
    if (!as_query) {
        const uint32_t t = tf[i];
        if (out_tf) out_tf[base + i] = t;
        atomicAdd((unsigned long long *)&len[v], (unsigned long long)t);
        if (t == 0) atomicMin(&flags[0], v);
        if (t >= (1u << 24)) atomicMin(&flags[1], v);
    }
    if (out_ord) {
        const uint32_t t = key_rank(vocab, T, kk);
        out_ord[base + i] = t < T && vocab[t] == kk ? t : BM25X_TERM_MISSING;
    }
}

// One thread per element of a document cast: the keys the vocabulary lacks (ord == BM25X_TERM_MISSING) as Key128,
// appended at out[atomicAdd(n)] in any order (a sort follows); out == NULL counts them only.
__global__ void k_tsv_missing(const ulonglong2 *__restrict__ key, const uint32_t *__restrict__ ord, uint64_t E,
                              Key128 *__restrict__ out, uint32_t *__restrict__ n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool miss = i < E && ord[i] == BM25X_TERM_MISSING;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, miss);
    if (!b) return;
    const uint32_t lane = threadIdx.x & 31, leader = __ffs(b) - 1;
    uint32_t at = 0;
    if (lane == leader) at = atomicAdd(n, (uint32_t)__popc(b));
    at = __shfl_sync(0xFFFFFFFFu, at, leader);
    if (miss && out) out[at + __popc(b & ((1u << lane) - 1u))] = key_of(key[i]);
}

// One thread per element: a key the vocabulary lacks takes uord[its rank in u[0..nu)], the call's distinct missing keys
// ascending.
__global__ void k_tsv_fresh(const ulonglong2 *__restrict__ key, uint32_t *__restrict__ ord, uint64_t E,
                            const Key128 *__restrict__ u, uint32_t nu, const uint32_t *__restrict__ uord) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E || ord[i] != BM25X_TERM_MISSING) return;
    ord[i] = uord[key_rank(u, nu, key_of(key[i]))];
}

}  // namespace

// Every refusal of a batch of tsvectors that needs only the host (TsVectorBorrowed::iter's panics, tsvector.rs:55-71,
// and "tsvector must have positions", tsvector.rs:88), named by who.
int check_tsvectors(const char *who, const bm25x_tsvectors *t, int as_query) {
    if (!t->ent_off || !t->byte_off) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    const uint32_t n = t->n;
    if (t->ent_off[0] != 0 || t->byte_off[0] != 0) {
        bm25x_set_error("%s: invalid data: ent_off[0] and byte_off[0] must be 0", who);
        return BM25X_ERR_INVALID;
    }
    for (uint32_t v = 0; v < n; v++)  // before any entry is read: the ranges must lie inside the arrays
        if (t->ent_off[v + 1] < t->ent_off[v] || t->byte_off[v + 1] < t->byte_off[v]) {
            bm25x_set_error("%s: invalid data: offsets not monotone at tsvector %u", who, v);
            return BM25X_ERR_INVALID;
        }
    if ((!t->entries && t->ent_off[n]) || (!t->bytes && t->byte_off[n])) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    // per vector: 0 = valid, else 1 + the fault (1 lexeme past the area, 2 count past the area, 3 no positions) and the
    // entry (index inside the vector)
    auto fault = [&](uint32_t v, uint64_t *entry) {
        const uint64_t size = t->byte_off[v + 1] - t->byte_off[v];
        for (uint64_t j = t->ent_off[v]; j < t->ent_off[v + 1]; j++) {
            const uint32_t e = t->entries[j], len = (e >> 1) & 0x7FFu, pos = e >> 12;
            *entry = j - t->ent_off[v];
            if ((uint64_t)pos + len > size) return 1;
            if (e & 1u) {
                if ((((uint64_t)pos + len + 1) & ~1ull) + 2 > size) return 2;
            } else if (!as_query) {
                return 3;
            }
        }
        return 0;
    };
    uint32_t first = 0xFFFFFFFFu;
#pragma omp parallel for schedule(dynamic, 1024) reduction(min : first) num_threads(bm25x_host_threads(0))
    for (uint32_t v = 0; v < n; v++) {
        uint64_t j;
        if (fault(v, &j)) first = std::min(first, v);
    }
    if (first == 0xFFFFFFFFu) return BM25X_OK;
    uint64_t j = 0;
    const int f = fault(first, &j);
    const unsigned long long jj = (unsigned long long)j;
    if (f == 1) bm25x_set_error("%s: invalid data: the lexeme of entry %llu of tsvector %u runs past its area", who, jj, first);
    else if (f == 2)
        bm25x_set_error("%s: invalid data: the position count of entry %llu of tsvector %u runs past its area", who, jj, first);
    else bm25x_set_error("%s: invalid data: tsvector must have positions (entry %llu of tsvector %u)", who, jj, first);
    return BM25X_ERR_INVALID;
}

namespace {

// Document::new (vector.rs:51-64): an element of value 0 is invalid data; v numbers the vector in the caller's batch.
int zero_refusal(const char *who, uint32_t v) {
    bm25x_set_error("%s: invalid data: a lexeme of tsvector %u has position counts that sum to 0", who, v);
    return BM25X_ERR_INVALID;
}

// The refusal of a merged tf the packed posting layout cannot hold, naming the document.
int big_tf_refusal(const char *who, uint32_t d) {
    bm25x_set_error("%s: term frequency >= 2^24 is not supported by the packed posting layout (document %u)", who, d);
    return BM25X_ERR_UNSUPPORTED;
}

int run_cast(const char *who, const bm25x_tsvectors *t, const uint8_t seed[32], int as_query, bool want_keys,
             const Key128 *vocab, uint32_t T, TsvCast &c) {
    Scratch &sc = c.sc;
    const uint32_t n = t->n;
    // entries and bytes are read at the absolute offsets ent_off / byte_off give, so that a slice of a batch (its
    // offsets + lo, entries and bytes as they are) casts in place; its outputs hold its own entries only
    const uint64_t E = t->ent_off[n] - t->ent_off[0];
    // the chunks: whole vectors, at most CHUNK_ENT entries, CHUNK_BYTES bytes and CHUNK_VEC vectors, or one vector
    std::vector<uint32_t> cuts{0};
    while (cuts.back() < n) {
        const uint32_t a = cuts.back();
        uint32_t b = a + 1;
        while (b < n && b - a < CHUNK_VEC && t->ent_off[b + 1] - t->ent_off[a] <= CHUNK_ENT &&
               t->byte_off[b + 1] - t->byte_off[a] <= CHUNK_BYTES)
            b++;
        cuts.push_back(b);
    }
    uint64_t ce = 0, cb = 0, cv = 0;
    for (size_t k = 0; k + 1 < cuts.size(); k++) {
        ce = std::max(ce, t->ent_off[cuts[k + 1]] - t->ent_off[cuts[k]]);
        cb = std::max(cb, t->byte_off[cuts[k + 1]] - t->byte_off[cuts[k]]);
        cv = std::max<uint64_t>(cv, cuts[k + 1] - cuts[k]);
    }
    if (ce > 0x7FFFFFFFull) {
        bm25x_set_error("%s: a tsvector of %llu entries, more than the 2^31 - 1 one sort takes", who,
                        (unsigned long long)ce);
        return BM25X_ERR_UNSUPPORTED;
    }
    Seed sd;
    for (int i = 0; i < 8; i++)
        sd.w[i] = (uint32_t)seed[4 * i] | (uint32_t)seed[4 * i + 1] << 8 | (uint32_t)seed[4 * i + 2] << 16 |
                  (uint32_t)seed[4 * i + 3] << 24;
    sc.e = cudaSetDevice(sc.device);
    if (want_keys) c.key = sc.alloc<ulonglong2>(E);
    if (!as_query) c.tf = sc.alloc<uint32_t>(E);
    if (vocab) c.ord = sc.alloc<uint32_t>(E);
    uint32_t *rows = sc.alloc<uint32_t>(n), *flags = sc.alloc<uint32_t>(2);
    uint64_t *len = as_query ? nullptr : sc.alloc<uint64_t>(n);
    Scratch tmp(sc.device);  // the chunk buffers, freed before the caller goes on
    uint32_t *d_ent = tmp.alloc<uint32_t>(ce), *cnt[2] = {tmp.alloc<uint32_t>(ce), tmp.alloc<uint32_t>(ce)};
    uint8_t *d_bytes = tmp.alloc<uint8_t>(cb);
    uint64_t *d_eoff = tmp.alloc<uint64_t>(cv + 1), *d_boff = tmp.alloc<uint64_t>(cv + 1);
    VKey *key[2] = {tmp.alloc<VKey>(ce), tmp.alloc<VKey>(ce)};
    int64_t *d_runs = tmp.alloc<int64_t>(1);
    size_t sort_bytes = 0, red_bytes = 0;
    if (tmp.e == cudaSuccess && ce) {
        cub::DoubleBuffer<VKey> k(key[0], key[1]);
        cub::DoubleBuffer<uint32_t> v(cnt[0], cnt[1]);
        tmp.e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, k, v, (int)ce, VKeyBits{}, 0, 160);
        if (tmp.e == cudaSuccess)
            tmp.e = cub::DeviceReduce::ReduceByKey(nullptr, red_bytes, key[0], key[1], cnt[0], cnt[1], d_runs, SatAdd{},
                                                   (int)ce);
    }
    void *temp = tmp.alloc<uint8_t>(std::max(sort_bytes, red_bytes));
    if (sc.e == cudaSuccess) sc.e = tmp.e;
    if (sc.e == cudaSuccess) sc.e = cudaMemset(rows, 0, sizeof(uint32_t) * (size_t)n);
    if (sc.e == cudaSuccess) sc.e = cudaMemset(flags, 0xFF, 2 * sizeof(uint32_t));
    if (sc.e == cudaSuccess && len) sc.e = cudaMemset(len, 0, sizeof(uint64_t) * (size_t)n);
    std::vector<uint64_t> h_eoff, h_boff;
    uint64_t base = 0;
    for (size_t k = 0; k + 1 < cuts.size() && sc.e == cudaSuccess; k++) {
        const uint32_t a = cuts[k], b = cuts[k + 1], nv = b - a;
        const uint64_t e0 = t->ent_off[a], ne = t->ent_off[b] - e0, b0 = t->byte_off[a], nb = t->byte_off[b] - b0;
        if (ne == 0) continue;
        h_eoff.resize(nv + 1);
        h_boff.resize(nv + 1);
        for (uint32_t u = 0; u <= nv; u++) {
            h_eoff[u] = t->ent_off[a + u] - e0;
            h_boff[u] = t->byte_off[a + u] - b0;
        }
        sc.e = cudaMemcpy(d_ent, t->entries + e0, sizeof(uint32_t) * ne, cudaMemcpyHostToDevice);
        if (sc.e == cudaSuccess && nb) sc.e = cudaMemcpy(d_bytes, t->bytes + b0, nb, cudaMemcpyHostToDevice);
        if (sc.e == cudaSuccess) sc.e = cudaMemcpy(d_eoff, h_eoff.data(), sizeof(uint64_t) * (nv + 1), cudaMemcpyHostToDevice);
        if (sc.e == cudaSuccess) sc.e = cudaMemcpy(d_boff, h_boff.data(), sizeof(uint64_t) * (nv + 1), cudaMemcpyHostToDevice);
        if (sc.e != cudaSuccess) break;
        k_tsv_intern<<<grid_of(ne), TPB>>>(d_ent, ne, d_eoff, d_boff, nv, d_bytes, sd, as_query, key[0], cnt[0]);
        if (as_query) sc.e = cudaMemsetAsync(cnt[0], 0, sizeof(uint32_t) * ne);  // no counts: the merge still needs values
        if (sc.e == cudaSuccess) sc.e = cudaGetLastError();
        const int vbits = nv > 1 ? 32 - __builtin_clz(nv - 1) : 1;
        cub::DoubleBuffer<VKey> kd(key[0], key[1]);
        cub::DoubleBuffer<uint32_t> vd(cnt[0], cnt[1]);
        if (sc.e == cudaSuccess)
            sc.e = cub::DeviceRadixSort::SortPairs(temp, sort_bytes, kd, vd, (int)ne, VKeyBits{}, 0, 128 + vbits);
        VKey *ko = kd.Alternate();
        uint32_t *vo = vd.Alternate();
        if (sc.e == cudaSuccess)
            sc.e = cub::DeviceReduce::ReduceByKey(temp, red_bytes, kd.Current(), ko, vd.Current(), vo, d_runs, SatAdd{},
                                                  (int)ne);
        if (sc.e == cudaSuccess) {
            k_tsv_emit<<<grid_of(ne), TPB>>>(ko, vo, d_runs, a, base, as_query, c.key, c.tf, vocab, T, c.ord, rows, len,
                                             flags);
            sc.e = cudaGetLastError();
        }
        int64_t runs = 0;
        if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&runs, d_runs, sizeof(runs), cudaMemcpyDeviceToHost);
        base += (uint64_t)runs;
    }
    std::vector<uint32_t> h_rows(n);
    if (sc.e == cudaSuccess && n) sc.e = cudaMemcpy(h_rows.data(), rows, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost);
    uint32_t h_flags[2] = {0xFFFFFFFFu, 0xFFFFFFFFu};
    if (sc.e == cudaSuccess) sc.e = cudaMemcpy(h_flags, flags, sizeof(h_flags), cudaMemcpyDeviceToHost);
    std::vector<uint64_t> h_len(len ? n : 0);
    if (sc.e == cudaSuccess && len && n) sc.e = cudaMemcpy(h_len.data(), len, sizeof(uint64_t) * n, cudaMemcpyDeviceToHost);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "tsvector cast", sc.e);
    c.off.assign((size_t)n + 1, 0);
    for (uint32_t v = 0; v < n; v++) c.off[v + 1] = c.off[v] + h_rows[v];
    c.len.resize(h_len.size());
    for (size_t v = 0; v < h_len.size(); v++) c.len[v] = (uint32_t)std::min<uint64_t>(h_len[v], 0xFFFFFFFFu);
    c.zero = h_flags[0];
    c.big = h_flags[1];
    return c.zero != 0xFFFFFFFFu ? zero_refusal(who, c.zero) : BM25X_OK;
}

bool null_seed_or_tsv(const char *who, const bm25x_tsvectors *t, const uint8_t *seed) {
    if (t && seed) return false;
    bm25x_set_error("%s: null argument", who);
    return true;
}

// v's vocabulary as Key128 on v.device, uploaded on first use and kept in *v.slot by its owner.  Leaves v.device current.
int device_vocab(const char *who, const TsvVocab &v, const Key128 **out) {
    cudaError_t e = cudaSetDevice(v.device);
    if (e != cudaSuccess) return cuda_refusal(who, "vocabulary upload", e);
    std::lock_guard<std::mutex> lk(*v.mu);
    if (!*v.slot) {
        Scratch s(v.device);
        Key128 *p = upload_vocab(s, *v.keys, v.T);
        if (s.e == cudaSuccess) s.e = cudaDeviceSynchronize();
        if (s.e != cudaSuccess) return cuda_refusal(who, "vocabulary upload", s.e);
        *v.slot = s.release(p);
    }
    *out = (const Key128 *)*v.slot;
    return BM25X_OK;
}

}  // namespace

int tsvector_cast(const char *who, const TsvVocab &v, const uint8_t seed[32], const bm25x_tsvectors *t, int as_query,
                  TsvCast &c) {
    const Key128 *vocab = nullptr;
    const int rc = device_vocab(who, v, &vocab);
    return rc == BM25X_OK ? run_cast(who, t, seed, as_query, false, vocab, v.T, c) : rc;
}

int tsvector_rows(const char *who, const TsvVocab &v, const uint8_t seed[32], const bm25x_tsvectors *t, int as_query,
                  const TsvNumbering &number, TsvRows &out) {
    const Key128 *vocab = nullptr;
    int rc = device_vocab(who, v, &vocab);
    if (rc != BM25X_OK) return rc;
    TsvCast c(v.device);
    rc = run_cast(who, t, seed, as_query, !as_query, vocab, v.T, c);
    if (rc != BM25X_OK) return rc;
    const uint32_t n = t->n;
    const uint64_t E = c.off[n];
    Scratch &sc = c.sc;
    uint32_t *ord = c.ord, *tf = c.tf;
    if (!as_query) {
        if (E > 0x7FFFFFFFull || n > 0x7FFFFFFFu) {  // the sorts below take int sizes
            bm25x_set_error("%s: %llu elements in %u tsvectors, more than the 2^31 - 1 one insert sorts", who,
                            (unsigned long long)E, n);
            return BM25X_ERR_UNSUPPORTED;
        }
        // ---- the keys the vocabulary lacks: compacted, sorted and made distinct (U) ----
        uint32_t *d_m = sc.alloc<uint32_t>(2), M = 0;
        if (sc.e == cudaSuccess) sc.e = cudaMemset(d_m, 0, 2 * sizeof(uint32_t));
        if (sc.e == cudaSuccess && E) {
            k_tsv_missing<<<grid_of(E), TPB>>>(c.key, ord, E, nullptr, d_m);
            sc.e = cudaGetLastError();
        }
        if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&M, d_m, sizeof(M), cudaMemcpyDeviceToHost);
        if (sc.e == cudaSuccess && M) {
            Key128 *mk[2] = {sc.alloc<Key128>(M), sc.alloc<Key128>(M)};
            cub::DoubleBuffer<Key128> kb(mk[0], mk[1]);
            size_t sort_bytes = 0, uniq_bytes = 0;
            if (sc.e == cudaSuccess)
                sc.e = cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, kb, (int)M, Key128Bits{}, 0, 128);
            if (sc.e == cudaSuccess) sc.e = cub::DeviceSelect::Unique(nullptr, uniq_bytes, mk[0], mk[1], d_m + 1, M);
            void *temp = sc.alloc<uint8_t>(std::max(sort_bytes, uniq_bytes));
            if (sc.e == cudaSuccess) sc.e = cudaMemset(d_m, 0, sizeof(uint32_t));
            if (sc.e == cudaSuccess) {
                k_tsv_missing<<<grid_of(E), TPB>>>(c.key, ord, E, mk[0], d_m);
                sc.e = cudaGetLastError();
            }
            if (sc.e == cudaSuccess) sc.e = cub::DeviceRadixSort::SortKeys(temp, sort_bytes, kb, (int)M, Key128Bits{}, 0, 128);
            Key128 *u = kb.Alternate();
            if (sc.e == cudaSuccess) sc.e = cub::DeviceSelect::Unique(temp, uniq_bytes, kb.Current(), u, d_m + 1, M);
            uint32_t nu = 0;
            if (sc.e == cudaSuccess) sc.e = cudaMemcpy(&nu, d_m + 1, sizeof(nu), cudaMemcpyDeviceToHost);
            std::vector<Key128> h_u(nu);
            if (sc.e == cudaSuccess) sc.e = cudaMemcpy(h_u.data(), u, sizeof(Key128) * nu, cudaMemcpyDeviceToHost);
            if (sc.e != cudaSuccess) return cuda_refusal(who, "tsvector cast", sc.e);
            // ---- their ordinals, from the caller ----
            std::vector<uint8_t> raw((size_t)nu * 16);
            for (uint32_t i = 0; i < nu; i++) {
                const ulonglong2 r = raw_of(h_u[i]);
                memcpy(&raw[(size_t)i * 16], &r, 16);
            }
            std::vector<uint32_t> uord(nu);
            rc = number(nu, raw.data(), uord.data());
            if (rc != BM25X_OK) return rc;
            const uint32_t *d_uord = sc.up(uord.data(), nu);
            if (sc.e == cudaSuccess) {
                k_tsv_fresh<<<grid_of(E), TPB>>>(c.key, ord, E, u, nu, d_uord);
                sc.e = cudaGetLastError();
            }
            // ---- each row re-sorted by ordinal (only rows with a missing key can be out of order) ----
            const uint64_t *d_off = sc.up(c.off.data(), (size_t)n + 1);
            uint32_t *ord2 = sc.alloc<uint32_t>(E), *tf2 = sc.alloc<uint32_t>(E);
            size_t seg_bytes = 0;
            if (sc.e == cudaSuccess)
                sc.e = cub::DeviceSegmentedSort::SortPairs(nullptr, seg_bytes, ord, ord2, tf, tf2, (int)E, (int)n, d_off,
                                                          d_off + 1);
            void *seg_temp = sc.alloc<uint8_t>(seg_bytes);
            if (sc.e == cudaSuccess)
                sc.e = cub::DeviceSegmentedSort::SortPairs(seg_temp, seg_bytes, ord, ord2, tf, tf2, (int)E, (int)n, d_off,
                                                          d_off + 1);
            ord = ord2;
            tf = tf2;
        }
        out.tf.resize(E);
        if (sc.e == cudaSuccess && E) sc.e = cudaMemcpy(out.tf.data(), tf, sizeof(uint32_t) * E, cudaMemcpyDeviceToHost);
        out.len = std::move(c.len);
    }
    out.ord.resize(E);
    if (sc.e == cudaSuccess && E) sc.e = cudaMemcpy(out.ord.data(), ord, sizeof(uint32_t) * E, cudaMemcpyDeviceToHost);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "tsvector cast", sc.e);
    out.off = std::move(c.off);
    return BM25X_OK;
}

extern "C" int bm25x_cast_tsvectors(const bm25x_tsvectors *tsv, const uint8_t seed[32], int as_query, int device,
                                    uint64_t *out_off, uint8_t *out_key, uint32_t *out_tf) {
    const char *who = "bm25x_cast_tsvectors";
    if (null_seed_or_tsv(who, tsv, seed)) return BM25X_ERR_INVALID;
    if (!out_off || !out_key || (!as_query && !out_tf)) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_tsvectors(who, tsv, as_query);
    if (rc == BM25X_OK) rc = check_device(who, device);
    if (rc != BM25X_OK) return rc;
    TsvCast c(device);
    rc = run_cast(who, tsv, seed, as_query, true, nullptr, 0, c);
    if (rc != BM25X_OK) return rc;
    const uint64_t E = c.off[tsv->n];
    cudaError_t e = cudaSuccess;
    if (E) e = cudaMemcpy(out_key, c.key, 16 * E, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && E && !as_query) e = cudaMemcpy(out_tf, c.tf, sizeof(uint32_t) * E, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return cuda_refusal(who, "tsvector cast", e);
    memcpy(out_off, c.off.data(), sizeof(uint64_t) * c.off.size());
    return BM25X_OK;
}

extern "C" int bm25x_index_create_from_tsvectors(const bm25x_tsvectors *tsv, const uint8_t seed[32],
                                                 const uint16_t *payload, double k1, double b, int device,
                                                 bm25x_index **out) {
    const char *who = "bm25x_index_create_from_tsvectors";
    if (out) *out = nullptr;
    if (null_seed_or_tsv(who, tsv, seed) || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_tsvectors(who, tsv, 0);
    if (rc == BM25X_OK) rc = check_common(who, tsv->n, tsv->ent_off, k1, b, 0);
    if (rc != BM25X_OK && rc != BM25X_ERR_CUDA) return rc;
    rc = check_device(who, device);
    if (rc != BM25X_OK) return rc;
    TsvCast c(device);
    rc = run_cast(who, tsv, seed, 0, true, nullptr, 0, c);
    if (rc != BM25X_OK) return rc;
    if (c.big != 0xFFFFFFFFu) return big_tf_refusal(who, c.big);
    // the keyed documents of the cast, on the device: ascending keys and non-zero tf by construction
    bm25x_documents d{};
    d.n_docs = tsv->n;
    d.elem_off = c.off.data();
    d.elem_key = reinterpret_cast<const uint8_t *>(c.key);
    d.elem_tf = c.tf;
    d.payload = payload;
    d.k1 = k1;
    d.b = b;
    return documents_build(who, &d, c.len.data(), device, out);
}

// The sharded build from tsvectors: every shard's slice cast on its own device, one vocabulary merged on the host from
// the shards' distinct keys, each shard's keys turned into that vocabulary's ordinals, then the shards built one after
// the other from (ordinal, tf) alone.  A shard's keys never leave its device; only its distinct keys and their counts do.
extern "C" int bm25x_index_create_sharded_from_tsvectors(const bm25x_tsvectors *tsv, const uint8_t seed[32],
                                                         const uint16_t *payload, double k1, double b, uint32_t S,
                                                         const uint32_t *doc_bounds, const int *devices,
                                                         bm25x_sharded_index **out) {
    const char *who = "bm25x_index_create_sharded_from_tsvectors";
    if (out) *out = nullptr;
    if (null_seed_or_tsv(who, tsv, seed) || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    // every host check before any device is used: the tsvectors and the build's arguments as
    // bm25x_index_create_from_tsvectors checks them, then the shard arguments as bm25x_sharded_create checks them
    int rc = check_tsvectors(who, tsv, 0);
    if (rc == BM25X_OK) rc = check_common(who, tsv->n, tsv->ent_off, k1, b, 0);
    if (rc != BM25X_OK && rc != BM25X_ERR_CUDA) return rc;
    const uint32_t N = tsv->n;
    rc = check_shard_args(N, S, doc_bounds);
    if (rc != BM25X_OK) return rc;
    struct {
        uint32_t n_docs, n_terms;
        double k1, b;
    } seg{N, 0, k1, b};  // n_terms: the merged vocabulary's size once prepare has run
    uint64_t P = 0;
    std::vector<uint8_t> keys;                       // the segment's vocabulary, 16 B per key
    std::vector<uint32_t> df, len(N);                // the segment's df; each document's length (the cast's row sums)
    std::vector<std::unique_ptr<TsvCast>> cast(S);   // shard s's cast: keyed, then (ordinals written) ord + tf
    std::vector<std::vector<uint32_t>> df_s(S);      // shard s's df over the segment's vocabulary
    Stats st(N, 0, nullptr, 0, k1, b);
    auto prepare = [&](int, std::vector<uint64_t> *cum) {
        std::vector<uint64_t> ent(tsv->ent_off, tsv->ent_off + (size_t)N + 1);  // c_d = the entries of tsvector d
        const std::vector<uint32_t> bounds = shard_bounds(doc_bounds, ent, N, S);
        // ---- every shard's slice cast on its device; refused only once every shard is cast, in the unsharded order ----
        uint32_t zero = 0xFFFFFFFFu, big = 0xFFFFFFFFu;  // the first such vector, global numbering
        for (uint32_t s = 0; s < S; s++) {
            const uint32_t lo = bounds[s], hi = bounds[s + 1];
            // the slice: run_cast reads entries and bytes at the offsets ent_off / byte_off give, so only those move
            const bm25x_tsvectors t{hi - lo, tsv->ent_off + lo, tsv->entries, tsv->byte_off + lo, tsv->bytes};
            cast[s].reset(new TsvCast(devices ? devices[s] : 0));
            TsvCast &c = *cast[s];
            const int rc = run_cast(who, &t, seed, 0, true, nullptr, 0, c);
            if (rc != BM25X_OK && c.zero == 0xFFFFFFFFu) return rc;
            if (rc != BM25X_OK || c.big != 0xFFFFFFFFu) {
                if (c.zero != 0xFFFFFFFFu) zero = std::min(zero, lo + c.zero);
                else big = std::min(big, lo + c.big);
                cast[s].reset();
                continue;
            }
            std::copy(c.len.begin(), c.len.end(), len.begin() + lo);
            std::vector<uint32_t>().swap(c.len);
        }
        if (zero != 0xFFFFFFFFu) return zero_refusal(who, zero);
        if (big != 0xFFFFFFFFu) return big_tf_refusal(who, big);
        // ---- per shard, on its device: its distinct keys and their counts ----
        std::vector<std::vector<uint8_t>> keys_s(S);
        std::vector<std::vector<uint32_t>> cnt_s(S);
        size_t total = 0;
        for (uint32_t s = 0; s < S; s++) {
            const TsvCast &c = *cast[s];
            bm25x_documents d{};  // the slice's device-resident keyed CSR
            d.n_docs = bounds[s + 1] - bounds[s];
            d.elem_off = c.off.data();
            d.elem_key = reinterpret_cast<const uint8_t *>(c.key);
            d.elem_tf = c.tf;
            const int rc = vocab_pass(who, &d, c.sc.device, keys_s[s], cnt_s[s]);
            if (rc != BM25X_OK) return rc;
            total += cnt_s[s].size();
        }
        // ---- the segment's vocabulary: the shards' ascending key lists merged (a heap of the S list heads), each
        // shard key's global ordinal noted as it is taken ----
        std::vector<size_t> at(S, 0);  // the next key of each list
        std::vector<std::vector<uint32_t>> ord_s(S);
        auto later = [&](uint32_t a, uint32_t b) {
            const int c = memcmp(&keys_s[a][16 * at[a]], &keys_s[b][16 * at[b]], 16);
            return c > 0 || (c == 0 && a > b);
        };
        std::priority_queue<uint32_t, std::vector<uint32_t>, decltype(later)> heads(later);
        for (uint32_t s = 0; s < S; s++) {
            ord_s[s].resize(cnt_s[s].size());
            if (!cnt_s[s].empty()) heads.push(s);
        }
        keys.clear();
        keys.reserve(16 * total);  // at most every shard's keys, distinct
        while (!heads.empty()) {
            const uint32_t s = heads.top();
            heads.pop();
            const uint8_t *k = &keys_s[s][16 * at[s]];
            if (keys.empty() || memcmp(&keys[keys.size() - 16], k, 16) != 0) keys.insert(keys.end(), k, k + 16);
            ord_s[s][at[s]] = (uint32_t)std::min<uint64_t>(keys.size() / 16 - 1, 0xFFFFFFFFull);
            if (++at[s] < cnt_s[s].size()) heads.push(s);
        }
        std::vector<std::vector<uint8_t>>().swap(keys_s);
        keys.shrink_to_fit();
        const uint64_t V = keys.size() / 16;
        if (V > 0xFFFFFFFEull) {  // vocab_pass's refusal
            bm25x_set_error("%s: %llu distinct keys, more than the 2^32 - 2 term ordinals", who, (unsigned long long)V);
            return BM25X_ERR_UNSUPPORTED;
        }
        const uint32_t T = (uint32_t)V;
        // ---- each shard's counts at their global ordinals: its df; summed, the segment's ----
        df.assign(T, 0);
        for (uint32_t s = 0; s < S; s++) {
            df_s[s].assign(T, 0);
            for (size_t i = 0; i < cnt_s[s].size(); i++) {
                df_s[s][ord_s[s][i]] = cnt_s[s][i];
                df[ord_s[s][i]] += cnt_s[s][i];
            }
            std::vector<uint32_t>().swap(cnt_s[s]);
            std::vector<uint32_t>().swap(ord_s[s]);
        }
        seg.n_terms = T;
        st = Stats(N, doc_norms(N, len.data(), nullptr, 0, nullptr), df.data(), T, k1, b);
        // ---- per shard, its keys as ordinals of the vocabulary; the keys freed ----
        for (uint32_t s = 0; s < S; s++) {
            TsvCast &c = *cast[s];
            const uint64_t E = c.off.back();
            P += E;
            c.ord = c.sc.alloc<uint32_t>(E);
            cudaError_t e = c.sc.e;
            if (e == cudaSuccess && E) e = key_ordinals(c.sc.device, c.key, E, keys, T, c.ord);
            if (e == cudaSuccess) e = cudaSetDevice(c.sc.device);
            if (e == cudaSuccess) e = cudaFree(c.sc.release(c.key));
            if (e != cudaSuccess) return cuda_refusal(who, "key ordinals", e);
            c.key = nullptr;
        }
        if (cum) cum->swap(ent);
        return BM25X_OK;
    };
    // one shard at a time, from its ordinals and tf; the term keys once, with shard 0
    auto build = [&](uint32_t s, int device, uint32_t lo, uint32_t hi, IndexGuard &ix) {
        TsvCast &c = *cast[s];
        const uint32_t n = hi - lo, T = seg.n_terms;
        BuildMeta m{n, T, len.data() + lo, payload ? payload + (size_t)lo * 3 : nullptr, s ? nullptr : keys.data(), k1, b,
                    df_s[s].data(), c.off[n]};
        m.doc_base = lo;
        bm25x_documents d{};  // keyless: the cast's ordinals and tf, on the shard's device
        d.n_docs = n;
        d.elem_off = c.off.data();
        d.elem_term = c.ord;
        d.elem_tf = c.tf;
        d.n_terms = T;
        d.k1 = k1;
        d.b = b;
        int rc = index_begin(m, &st, device, ix);
        if (rc == BM25X_OK) rc = invert(who, &d, keys, 0, n, ix.get());
        cast[s].reset();
        std::vector<uint32_t>().swap(df_s[s]);
        return rc;
    };
    return sharded_build(who, &seg, P, df, st, S, doc_bounds, devices, prepare, build, out);
}

// Queries from tsvectors against the keys of ix (an index, or shard 0 of a document-sharded index, which holds the
// segment's keys), after the null checks; refusals named by who.
static int tsvector_queries(const char *who, bm25x_index *ix, const uint8_t seed[32], const bm25x_tsvectors *tsv,
                            uint32_t *q_off, uint32_t *q_terms) {
    int rc = check_tsvectors(who, tsv, 1);
    if (rc != BM25X_OK) return rc;
    if (!q_terms && tsv->ent_off[tsv->n]) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    const uint32_t T = ix->d.n_terms;
    if (ix->h_keys.empty() && T) {  // replicas and keyless builds: bm25x_lookup_terms' refusal
        bm25x_set_error("bm25x_lookup_terms: index was created without term keys");
        return BM25X_ERR_INVALID;
    }
    // the vocabulary as Key128, built once per handle and freed with it (bm25x_index_destroy)
    TsvCast c(ix->device);
    rc = tsvector_cast(who, {ix->device, &ix->h_keys, T, &ix->key_vocab, &ix->key_vocab_mutex}, seed, tsv, 1, c);
    if (rc != BM25X_OK) return rc;
    const uint64_t E = c.off[tsv->n];
    if (E > 0xFFFFFFFFull) {
        bm25x_set_error("%s: %llu query terms, more than the 2^32 - 1 that u32 offsets address", who,
                        (unsigned long long)E);
        return BM25X_ERR_UNSUPPORTED;
    }
    if (E) {
        const cudaError_t e = cudaMemcpy(q_terms, c.ord, sizeof(uint32_t) * E, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) return cuda_refusal(who, "tsvector cast", e);
    }
    for (uint32_t v = 0; v <= tsv->n; v++) q_off[v] = (uint32_t)c.off[v];
    return BM25X_OK;
}

extern "C" int bm25x_tsvector_queries(bm25x_index *ix, const uint8_t seed[32], const bm25x_tsvectors *tsv, uint32_t *q_off,
                                      uint32_t *q_terms) {
    const char *who = "bm25x_tsvector_queries";
    if (null_seed_or_tsv(who, tsv, seed) || !ix || !q_off) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    return tsvector_queries(who, ix, seed, tsv, q_off, q_terms);
}

extern "C" int bm25x_tsvector_queries_sharded(bm25x_sharded_index *sx, const uint8_t seed[32], const bm25x_tsvectors *tsv,
                                              uint32_t *q_off, uint32_t *q_terms) {
    const char *who = "bm25x_tsvector_queries_sharded";
    if (null_seed_or_tsv(who, tsv, seed) || !sx || !q_off) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    // shard 0 holds the segment's keys, and its handle the device copy of them (uploaded once, freed with the index)
    return tsvector_queries(who, sx->shards[0], seed, tsv, q_off, q_terms);
}
