// bm25x_documents.cu — an index built from documents (DESIGN §4.9): the inversion CREATE INDEX runs below the heap scan,
// on the GPU.
//
// The reference streams every row's Document (Element{key, value} sorted by key, crates/bm25/src/vector.rs:38-83) through
// io::write, which records Record(length, payload) and one Mapping(key, doc, tf) per element (crates/bm25/src/io.rs:187-197),
// sorts the mappings in 64 MiB runs on disk and k-way merges them (io.rs:69-98,199-244) into the Segment that
// bm25::build → flush takes.  Here the documents are read doc-major, in chunks of CHUNK elements (a chunk may cut a
// document: a term holds a document at most once and the chunks go in element order, which is doc order):
//   1. vocabulary and df.  Keyed: every chunk's keys as (big-endian hi, lo) u64 pairs, whose radix order is the bytewise
//      order, appended to a device list that is compacted (CUB radix sort + reduce by key) whenever the appended part
//      outgrows the compacted one; keyless: a df histogram of the ordinals;
//   2. the handle opened by index_begin, as the CSR build opens it (one Stats, the same padded offsets);
//   3. per chunk: the ordinals (keyed: each key found in the device vocabulary), a stable radix sort of (ordinal →
//      element) over ceil(log2 T) bits, and k_scatter writing {doc, tf << 8 | fieldnorm} at the term's padded offset +
//      the postings of the earlier chunks + the rank in the run; then index_finish_device.
// A document-sharded build counts every shard's df on the shard's device (the host sums them into the segment's), then
// inverts each shard's element range with local doc ids.
#include <string.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>

#include "bm25x_build.h"
#include "bm25x_keys.cuh"

namespace {

constexpr uint64_t CHUNK = 1ull << 22;  // elements per chunk

// Ordinal of each raw key of a chunk: its position in the sorted vocabulary (which holds every key of the documents);
// idx[i] = i when idx is given.
__global__ void k_key_ordinals(const ulonglong2 *__restrict__ raw, uint64_t n, const Key128 *__restrict__ vocab, uint32_t T,
                               uint32_t *__restrict__ term, uint32_t *__restrict__ idx) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    term[i] = key_rank(vocab, T, key_of(raw[i]));
    if (idx) idx[i] = (uint32_t)i;
}

__global__ void k_iota(uint32_t *__restrict__ idx, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (uint32_t)i;
}

// df += the elements of each ordinal; the lanes of a warp that share an ordinal add once.
__global__ void k_df_count(const uint32_t *__restrict__ term, uint64_t n, uint32_t *__restrict__ df) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n;
    const uint32_t t = live ? term[i] : 0xFFFFFFFFu;
    const uint32_t same = __match_any_sync(0xFFFFFFFFu, t);
    if (live && (threadIdx.x & 31) == (unsigned)(__ffs(same) - 1)) atomicAdd(&df[t], (uint32_t)__popc(same));
}

// At the first entry j of each ordinal's run in the sorted chunk: base[t] = where entry j's posting goes minus j (mod 2^64).
__global__ void k_run_heads(const uint32_t *__restrict__ term, uint64_t n, const uint64_t *__restrict__ post_off,
                            const uint32_t *__restrict__ cursor, uint64_t *__restrict__ base) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t t = term[j];
    if (j == 0 || term[j - 1] != t) base[t] = post_off[t] + cursor[t] - j;
}

// One thread per sorted entry j = (ordinal t, element i of the chunk that starts at element g0): the posting
// {doc, tf << 8 | fieldnorm[doc]} at base[t] + j (k_build_postings' packing); the last entry of the run moves the term's
// cursor past it.  doc = sdoc[k] for the last of the chunk's document starts start[0..n_start] (ascending, start[0] = g0)
// at or before element g0 + i.
__global__ void k_scatter(const uint32_t *__restrict__ term, const uint32_t *__restrict__ idx, uint64_t n, uint64_t g0,
                          const uint64_t *__restrict__ start, const uint32_t *__restrict__ sdoc, uint32_t n_start,
                          const uint32_t *__restrict__ tf, const uint64_t *__restrict__ base,
                          const uint64_t *__restrict__ post_off, const uint8_t *__restrict__ fieldnorm,
                          Posting *__restrict__ post, uint32_t *__restrict__ cursor) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t t = term[j], i = idx[j];
    const uint32_t d = sdoc[owner_of(start, n_start, g0 + i)];
    Posting p;
    p.doc = d;
    p.w = (tf[i] << 8) | fieldnorm[d];
    const uint64_t at = base[t] + j;
    post[at] = p;
    if (j + 1 == n || term[j + 1] != t) cursor[t] = (uint32_t)(at + 1 - post_off[t]);
}

// A device buffer that grows (keeping its first `keep` entries) and frees itself: the vocabulary pass's list.
template <typename T>
struct GrowBuf {
    T *p = nullptr;
    size_t cap = 0;
    GrowBuf() = default;
    GrowBuf(const GrowBuf &) = delete;
    ~GrowBuf() { cudaFree(p); }
    void swap(GrowBuf &o) {
        std::swap(p, o.p);
        std::swap(cap, o.cap);
    }
    cudaError_t grow(size_t n, size_t keep) {
        if (n <= cap) return cudaSuccess;
        T *q = nullptr;
        cudaError_t e = cudaMalloc((void **)&q, sizeof(T) * n);
        if (e == cudaSuccess && keep) e = cudaMemcpy(q, p, sizeof(T) * keep, cudaMemcpyDeviceToDevice);
        if (e != cudaSuccess) {
            cudaFree(q);
            return e;
        }
        cudaFree(p);
        p = q;
        cap = n;
        return cudaSuccess;
    }
};

// Ordinals of elements [g, g + n) into term: keyless as given; keyed the keys (copied to kbuf) looked up in the device
// vocabulary.  idx[i] = i when idx is given.  The element arrays may be host or device memory: the copies follow the
// addresses (a build from tsvectors hands its device-resident cast here).
cudaError_t load_ordinals(const bm25x_documents *c, uint64_t g, uint64_t n, const Key128 *vocab, uint32_t T,
                          ulonglong2 *kbuf, uint32_t *term, uint32_t *idx) {
    cudaError_t e;
    if (c->elem_key) {
        e = cudaMemcpy(kbuf, c->elem_key + g * 16, 16 * n, cudaMemcpyDefault);
        if (e != cudaSuccess) return e;
        k_key_ordinals<<<grid_of(n), TPB>>>(kbuf, n, vocab, T, term, idx);
        return cudaGetLastError();
    }
    e = cudaMemcpy(term, c->elem_term + g, sizeof(uint32_t) * n, cudaMemcpyDefault);
    if (e != cudaSuccess || !idx) return e;
    k_iota<<<grid_of(n), TPB>>>(idx, n);
    return cudaGetLastError();
}

}  // namespace

// Host pass over the documents, shared by both entry points: every refusal that needs no device (refusals named by
// bm25x_index_create_from_documents), and each document's length, the saturating Σ tf (Document::length,
// vector.rs:76-83).  The device check is the caller's.
static int validate_documents(const bm25x_documents *c, std::vector<uint32_t> &doc_len) {
    const char *who = "bm25x_index_create_from_documents";
    if (!c->elem_off || !c->elem_tf) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    if (!c->elem_key == !c->elem_term) {
        bm25x_set_error("%s: exactly one of elem_key and elem_term must be given", who);
        return BM25X_ERR_INVALID;
    }
    if (c->elem_key && c->n_terms) {
        bm25x_set_error("%s: n_terms must be 0 with elem_key (the keys make the vocabulary)", who);
        return BM25X_ERR_INVALID;
    }
    const int rc = check_common(who, c->n_docs, c->elem_off, c->k1, c->b, 0);
    if (rc != BM25X_OK && rc != BM25X_ERR_CUDA) return rc;
    const uint32_t N = c->n_docs;
    if (c->elem_off[0] != 0) {
        bm25x_set_error("%s: invalid data: elem_off[0] must be 0", who);
        return BM25X_ERR_INVALID;
    }
    for (uint32_t d = 0; d < N; d++)  // before any element is read: the ranges must lie inside [0, E)
        if (c->elem_off[d + 1] < c->elem_off[d]) {
            bm25x_set_error("%s: invalid data: offsets not monotone at document %u", who, d);
            return BM25X_ERR_INVALID;
        }
    // per document: 0 = valid, 1 = keys not ascending, 2 = ordinal >= n_terms, 3 = tf == 0, 4 = tf >= 2^24 (the others first)
    auto fault = [&](uint32_t d, uint32_t *len) {
        const uint64_t a = c->elem_off[d], e = c->elem_off[d + 1];
        uint64_t sum = 0;
        int f = 0;
        for (uint64_t i = a; i < e; i++) {
            const uint32_t tf = c->elem_tf[i];
            if (i > a && (c->elem_key ? memcmp(c->elem_key + (i - 1) * 16, c->elem_key + i * 16, 16) >= 0
                                      : c->elem_term[i - 1] >= c->elem_term[i]))
                return 1;
            if (c->elem_term && c->elem_term[i] >= c->n_terms) return 2;
            if (tf == 0) return 3;
            if (tf >= (1u << 24)) f = 4;
            sum += tf;
        }
        if (len) *len = (uint32_t)std::min<uint64_t>(sum, 0xFFFFFFFFu);
        return f;
    };
    doc_len.resize(N);
    uint32_t first_invalid = 0xFFFFFFFFu, first_unsupported = 0xFFFFFFFFu;
#pragma omp parallel for schedule(dynamic, 1024) reduction(min : first_invalid, first_unsupported) \
    num_threads(bm25x_host_threads(0))
    for (uint32_t d = 0; d < N; d++) {
        const int f = fault(d, &doc_len[d]);
        if (f == 4) first_unsupported = std::min(first_unsupported, d);
        else if (f) first_invalid = std::min(first_invalid, d);
    }
    if (first_invalid != 0xFFFFFFFFu) {
        const uint32_t d = first_invalid;
        switch (fault(d, nullptr)) {
        case 1: bm25x_set_error("%s: invalid data: keys of document %u are not strictly ascending", who, d); break;
        case 2: bm25x_set_error("%s: invalid data: a term ordinal of document %u is not below n_terms=%u", who, d, c->n_terms); break;
        default: bm25x_set_error("%s: invalid data: zero term frequency in document %u", who, d);
        }
        return BM25X_ERR_INVALID;
    }
    if (first_unsupported != 0xFFFFFFFFu) {
        bm25x_set_error("%s: term frequency >= 2^24 is not supported by the packed posting layout (document %u)", who,
                        first_unsupported);
        return BM25X_ERR_UNSUPPORTED;
    }
    return BM25X_OK;
}

// The vocabulary of a keyed build on `device`: the distinct keys of every element, ascending bytewise (host bytes), and
// each key's df.  Every chunk's keys are appended to a device list of (key, count); the list is compacted (sort by key,
// sum the counts of equal keys) when its appended part reaches its compacted part, so every entry is sorted a bounded
// number of times whatever the vocabulary's size.
int vocab_pass(const char *who, const bm25x_documents *c, int device, std::vector<uint8_t> &keys,
               std::vector<uint32_t> &df) {
    const uint64_t E = c->elem_off[c->n_docs];
    cudaError_t e = cudaSetDevice(device);
    GrowBuf<Key128> kb[2];
    GrowBuf<uint32_t> cb[2];
    GrowBuf<uint8_t> temp;
    Scratch sc(device);
    int64_t *d_runs = sc.alloc<int64_t>(1);
    if (e == cudaSuccess) e = sc.e;
    uint64_t V = 0, A = 0;  // compacted entries, then appended ones
    auto compact = [&]() -> cudaError_t {
        const int64_t n = (int64_t)(V + A);
        cub::DoubleBuffer<Key128> k(kb[0].p, kb[1].p);
        cub::DoubleBuffer<uint32_t> v(cb[0].p, cb[1].p);
        size_t sort_bytes = 0, red_bytes = 0;
        cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, k, v, n, Key128Bits{});
        if (e == cudaSuccess)
            e = cub::DeviceReduce::ReduceByKey(nullptr, red_bytes, k.Current(), k.Alternate(), v.Current(), v.Alternate(),
                                               d_runs, ::cuda::std::plus<uint32_t>{}, n);
        if (e == cudaSuccess) e = temp.grow(std::max(sort_bytes, red_bytes), 0);
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(temp.p, sort_bytes, k, v, n, Key128Bits{});
        if (e == cudaSuccess)
            e = cub::DeviceReduce::ReduceByKey(temp.p, red_bytes, k.Current(), k.Alternate(), v.Current(), v.Alternate(),
                                               d_runs, ::cuda::std::plus<uint32_t>{}, n);
        int64_t runs = 0;
        if (e == cudaSuccess) e = cudaMemcpy(&runs, d_runs, sizeof(runs), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) return e;
        if (k.Alternate() != kb[0].p) kb[0].swap(kb[1]);  // the reduced list is buffer 0
        if (v.Alternate() != cb[0].p) cb[0].swap(cb[1]);
        V = (uint64_t)runs;
        A = 0;
        return cudaSuccess;
    };
    for (uint64_t g = 0; g < E && e == cudaSuccess; g += CHUNK) {
        const uint64_t n = std::min(CHUNK, E - g);
        const size_t need = V + A + n;
        if (need > kb[0].cap) {
            const size_t cap = 2 * need;
            e = kb[0].grow(cap, V + A);
            if (e == cudaSuccess) e = cb[0].grow(cap, V + A);
            if (e == cudaSuccess) e = kb[1].grow(cap, 0);
            if (e == cudaSuccess) e = cb[1].grow(cap, 0);
            if (e != cudaSuccess) break;
        }
        e = cudaMemcpy(kb[0].p + V + A, c->elem_key + g * 16, 16 * n, cudaMemcpyDefault);
        if (e != cudaSuccess) break;
        k_keys_be<<<grid_of(n), TPB>>>(kb[0].p + V + A, cb[0].p + V + A, n);
        e = cudaGetLastError();
        A += n;
        if (e == cudaSuccess && (A >= std::max<uint64_t>(V, CHUNK) || g + n == E)) e = compact();
    }
    if (e != cudaSuccess) return cuda_refusal(who, "vocabulary pass", e);
    if (V > 0xFFFFFFFEull) {
        bm25x_set_error("%s: %llu distinct keys, more than the 2^32 - 2 term ordinals", who, (unsigned long long)V);
        return BM25X_ERR_UNSUPPORTED;
    }
    std::vector<Key128> h((size_t)V);
    df.resize(V);
    if (V) e = cudaMemcpy(h.data(), kb[0].p, sizeof(Key128) * V, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && V) e = cudaMemcpy(df.data(), cb[0].p, sizeof(uint32_t) * V, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return cuda_refusal(who, "vocabulary pass", e);
    keys.resize((size_t)V * 16);
    for (uint64_t t = 0; t < V; t++) {
        const ulonglong2 raw = raw_of(h[t]);
        memcpy(&keys[t * 16], &raw, 16);
    }
    return BM25X_OK;
}

// df of the T terms over elements [e0, e1), counted on `device` (keyed: each key looked up in the vocabulary first).
static int count_df(const char *who, const bm25x_documents *c, const std::vector<uint8_t> &keys, uint32_t T, uint64_t e0,
                    uint64_t e1, int device, std::vector<uint32_t> &df) {
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const uint64_t ch = std::min(CHUNK, e1 - e0);
    uint32_t *d_df = sc.alloc<uint32_t>(T), *d_term = sc.alloc<uint32_t>(ch);
    const Key128 *vocab = c->elem_key ? upload_vocab(sc, keys, T) : nullptr;
    ulonglong2 *kbuf = c->elem_key ? sc.alloc<ulonglong2>(ch) : nullptr;
    if (sc.e == cudaSuccess) sc.e = cudaMemset(d_df, 0, sizeof(uint32_t) * (size_t)T);
    for (uint64_t g = e0; g < e1 && sc.e == cudaSuccess; g += CHUNK) {
        const uint64_t n = std::min(CHUNK, e1 - g);
        sc.e = load_ordinals(c, g, n, vocab, T, kbuf, d_term, nullptr);
        if (sc.e == cudaSuccess) {
            k_df_count<<<grid_of(n), TPB>>>(d_term, n, d_df);
            sc.e = cudaGetLastError();
        }
    }
    df.resize(T);
    if (sc.e == cudaSuccess && T) sc.e = cudaMemcpy(df.data(), d_df, sizeof(uint32_t) * (size_t)T, cudaMemcpyDeviceToHost);
    return sc.e == cudaSuccess ? BM25X_OK : cuda_refusal(who, "df count", sc.e);
}

// The postings of documents [lo, hi) (local ids 0 .. hi - lo) written into the handle index_begin opened, chunk by chunk
// in element order; then index_finish_device.
int invert(const char *who, const bm25x_documents *c, const std::vector<uint8_t> &keys, uint32_t lo, uint32_t hi,
           bm25x_index *ix) {
    DeviceIndex &d = ix->d;
    const uint32_t T = d.n_terms;
    const uint64_t e0 = c->elem_off[lo], e1 = c->elem_off[hi], ch = std::min(CHUNK, e1 - e0);
    Scratch sc(ix->device);
    sc.e = cudaSetDevice(ix->device);
    // per chunk, its document starts: (element, local doc) of the document that holds its first element, then of every
    // non-empty document that begins inside it (at most one per element: the device memory does not grow with n_docs)
    std::vector<uint64_t> h_start;
    std::vector<uint32_t> h_sdoc;
    uint64_t *d_start = sc.alloc<uint64_t>(ch + 1);
    uint32_t *d_sdoc = sc.alloc<uint32_t>(ch + 1);
    uint32_t owner = lo;
    const Key128 *vocab = c->elem_key ? upload_vocab(sc, keys, T) : nullptr;
    ulonglong2 *kbuf = c->elem_key ? sc.alloc<ulonglong2>(ch) : nullptr;
    uint32_t *cursor = sc.alloc<uint32_t>(T);
    uint64_t *base = sc.alloc<uint64_t>(T);
    uint32_t *term[2] = {sc.alloc<uint32_t>(ch), sc.alloc<uint32_t>(ch)}, *idx[2] = {sc.alloc<uint32_t>(ch), sc.alloc<uint32_t>(ch)};
    uint32_t *d_tf = sc.alloc<uint32_t>(ch);
    const int bits = T > 1 ? 32 - __builtin_clz(T - 1) : 1;
    size_t temp_bytes = 0;
    void *temp = nullptr;
    if (sc.e == cudaSuccess) sc.e = cudaMemset(cursor, 0, sizeof(uint32_t) * (size_t)T);
    if (sc.e == cudaSuccess && ch) {
        cub::DoubleBuffer<uint32_t> k(term[0], term[1]), v(idx[0], idx[1]);
        sc.e = cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, k, v, (int)ch, 0, bits);
        temp = sc.alloc<uint8_t>(temp_bytes);
    }
    for (uint64_t g = e0; g < e1 && sc.e == cudaSuccess; g += CHUNK) {
        const uint64_t n = std::min(CHUNK, e1 - g);
        while (c->elem_off[owner + 1] <= g) owner++;
        h_start.assign(1, g);
        h_sdoc.assign(1, owner - lo);
        for (uint32_t doc = owner + 1; doc < hi && c->elem_off[doc] < g + n; doc++)
            if (c->elem_off[doc + 1] > c->elem_off[doc]) {
                h_start.push_back(c->elem_off[doc]);
                h_sdoc.push_back(doc - lo);
            }
        sc.e = load_ordinals(c, g, n, vocab, T, kbuf, term[0], idx[0]);
        if (sc.e == cudaSuccess) sc.e = cudaMemcpy(d_tf, c->elem_tf + g, sizeof(uint32_t) * n, cudaMemcpyDefault);
        if (sc.e == cudaSuccess)
            sc.e = cudaMemcpy(d_start, h_start.data(), sizeof(uint64_t) * h_start.size(), cudaMemcpyHostToDevice);
        if (sc.e == cudaSuccess)
            sc.e = cudaMemcpy(d_sdoc, h_sdoc.data(), sizeof(uint32_t) * h_sdoc.size(), cudaMemcpyHostToDevice);
        cub::DoubleBuffer<uint32_t> k(term[0], term[1]), v(idx[0], idx[1]);
        if (sc.e == cudaSuccess) sc.e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, k, v, (int)n, 0, bits);
        if (sc.e == cudaSuccess) {
            k_run_heads<<<grid_of(n), TPB>>>(k.Current(), n, d.post_off, cursor, base);
            k_scatter<<<grid_of(n), TPB>>>(k.Current(), v.Current(), n, g, d_start, d_sdoc, (uint32_t)h_start.size() - 1,
                                           d_tf, base, d.post_off, d.fieldnorm, d.post, cursor);
            sc.e = cudaGetLastError();
        }
    }
    if (sc.e == cudaSuccess) sc.e = cudaDeviceSynchronize();
    if (sc.e == cudaSuccess) sc.e = index_finish_device(ix);
    return sc.e == cudaSuccess ? BM25X_OK : cuda_refusal(who, "document inversion", sc.e);
}

cudaError_t key_ordinals(int device, const void *raw, uint64_t n, const std::vector<uint8_t> &keys, uint32_t T,
                         uint32_t *term) {
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const Key128 *vocab = upload_vocab(sc, keys, T);
    if (sc.e == cudaSuccess && n) {
        k_key_ordinals<<<grid_of(n), TPB>>>(static_cast<const ulonglong2 *>(raw), n, vocab, T, term, nullptr);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaDeviceSynchronize();
    return sc.e;
}

int documents_build(const char *who, const bm25x_documents *c, const uint32_t *doc_len, int device, bm25x_index **out) {
    const uint32_t N = c->n_docs;
    const uint64_t E = c->elem_off[N];
    std::vector<uint8_t> keys;
    std::vector<uint32_t> df;
    int rc = c->elem_key ? vocab_pass(who, c, device, keys, df) : count_df(who, c, keys, c->n_terms, 0, E, device, df);
    if (rc != BM25X_OK) return rc;
    const uint32_t T = (uint32_t)df.size();
    BuildMeta m{N, T, doc_len, c->payload, c->elem_key ? keys.data() : nullptr, c->k1, c->b, df.data(), E};
    IndexGuard ix;
    rc = index_begin(m, nullptr, device, ix);
    if (rc == BM25X_OK) rc = invert(who, c, keys, 0, N, ix.get());
    if (rc == BM25X_OK) *out = ix.release();
    return rc;
}

extern "C" int bm25x_index_create_from_documents(const bm25x_documents *c, int device, bm25x_index **out) {
    const char *who = "bm25x_index_create_from_documents";
    if (out) *out = nullptr;
    if (!c || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    std::vector<uint32_t> doc_len;
    int rc = validate_documents(c, doc_len);
    if (rc == BM25X_OK) rc = check_device(who, device);
    if (rc != BM25X_OK) return rc;
    return documents_build(who, c, doc_len.data(), device, out);
}

extern "C" int bm25x_index_create_sharded_from_documents(const bm25x_documents *c, uint32_t S, const uint32_t *doc_bounds,
                                                         const int *devices, bm25x_sharded_index **out) {
    const char *who = "bm25x_index_create_sharded_from_documents";
    if (out) *out = nullptr;
    if (!c || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    // every host check before any device is used: the documents as bm25x_index_create_from_documents checks them, then
    // the shard arguments as bm25x_sharded_create checks them
    std::vector<uint32_t> doc_len;
    int rc = validate_documents(c, doc_len);
    if (rc != BM25X_OK) return rc;
    const uint32_t N = c->n_docs;
    rc = check_shard_args(N, S, doc_bounds);
    if (rc != BM25X_OK) return rc;
    struct {
        uint32_t n_docs, n_terms;
        double k1, b;
    } seg{N, c->n_terms, c->k1, c->b};  // n_terms: a keyed build's vocabulary size once prepare has run
    const uint64_t sum_len = doc_norms(N, doc_len.data(), nullptr, 0, nullptr);
    std::vector<uint8_t> keys;
    std::vector<uint32_t> df;
    std::vector<std::vector<uint32_t>> df_s(S);
    Stats st(N, sum_len, nullptr, 0, c->k1, c->b);
    // the vocabulary on devices[0] (keyed), every shard's df on its own device, the segment's df and statistics
    auto prepare = [&](int dev0, std::vector<uint64_t> *cum) {
        if (c->elem_key) {
            const int rc = vocab_pass(who, c, dev0, keys, df);
            if (rc != BM25X_OK) return rc;
            seg.n_terms = (uint32_t)df.size();
        }
        const uint32_t T = seg.n_terms;
        std::vector<uint64_t> off(c->elem_off, c->elem_off + (size_t)N + 1);  // cum[d] = elem_off[d]: one posting per element
        const std::vector<uint32_t> bounds = shard_bounds(doc_bounds, off, N, S);
        df.assign(T, 0);
        for (uint32_t s = 0; s < S; s++) {
            const int rc = count_df(who, c, keys, T, off[bounds[s]], off[bounds[s + 1]], devices ? devices[s] : 0, df_s[s]);
            if (rc != BM25X_OK) return rc;
            for (uint32_t t = 0; t < T; t++) df[t] += df_s[s][t];
        }
        st = Stats(N, sum_len, df.data(), T, c->k1, c->b);
        if (cum) cum->swap(off);
        return BM25X_OK;
    };
    // one shard at a time, each inverting only its own elements; the term keys once, with shard 0
    auto build = [&](uint32_t s, int device, uint32_t lo, uint32_t hi, IndexGuard &ix) {
        BuildMeta m{hi - lo, seg.n_terms, doc_len.data() + lo, c->payload ? c->payload + (size_t)lo * 3 : nullptr,
                    s || !c->elem_key ? nullptr : keys.data(), c->k1, c->b, df_s[s].data(),
                    c->elem_off[hi] - c->elem_off[lo]};
        m.doc_base = lo;
        int rc = index_begin(m, &st, device, ix);
        if (rc == BM25X_OK) rc = invert(who, c, keys, lo, hi, ix.get());
        std::vector<uint32_t>().swap(df_s[s]);
        return rc;
    };
    return sharded_build(who, &seg, c->elem_off[N], df, st, S, doc_bounds, devices, prepare, build, out);
}
