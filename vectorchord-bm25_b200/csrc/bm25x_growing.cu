// bm25x_growing.cu — the growing segment (DESIGN §4.5): the one-shot handle of bm25x_growing_create, the mutable segment
// with its inserts, deletes, refresh and search, and the seal into a new sealed index.  Every handle is built by the
// contract of bm25x_build.h; the refresh and the seal splice with the kernels of bm25x_splice.cuh.  Tsvector inserts
// cast on the device (tsvector_rows, bm25x_tsvector.cu); the segment numbers the keys its sealed side lacks and hands
// them to its seal.
#include <string.h>

#include <algorithm>
#include <chrono>
#include <future>
#include <memory>
#include <unordered_map>
#include <unordered_set>

#include "bm25x_build.h"
#include "bm25x_splice.cuh"

// ---- f3: the growing segment (documents inserted since the last seal, search.rs:83-135) as a second, small index that
// scores with the sealed segment's statistics.  The reference scans these documents one by one per query; here they
// are inverted (term-major postings over growing ordinals) so that the same kernels unite them. ----

// Live postings of a batch of growing documents, term-major: the terms that hold any, ascending, and term[i]'s postings
// doc / tf[off[i] .. off[i + 1]) with ordinals ascending.
struct GrowingCsr {
    std::vector<uint32_t> term;
    std::vector<uint64_t> off{0};
    std::vector<uint32_t> doc, tf;
};

// The checks of growing documents (vector.rs:39-75: keys strictly ascending, tf != 0; tf < 2^24; every merged id below
// the BM25X_DOC_INF sentinel) and their inversion, for bm25x_growing_create and bm25x_growing_insert alike: the same codes
// and messages.  Document i becomes ordinal first + i; `first` growing documents already exist.  A deleted document, a
// BM25X_TERM_MISSING token and a term without sealed postings give no posting.
static int invert_growing(const SealedSide &sealed, const bm25x_growing_docs *g, uint32_t first, GrowingCsr &out) {
    const char *who = "bm25x_growing_create";
    const uint32_t G = g->n_docs, T = sealed.n_terms(), NS = sealed.n_docs();
    const std::vector<uint32_t> &sdf = sealed.df();
    if (!g->elem_off || (g->elem_off[G] && (!g->elem_term || !g->elem_tf))) {
        bm25x_set_error("%s: empty or malformed corpus", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_common(who, G, g->doc_len ? (const void *)g->doc_len : (const void *)g->doc_fieldnorm,
                          sealed.home().k1, sealed.home().b, sealed.home().device);
    if (rc != BM25X_OK) return rc;
    // growing documents come back as sealed n_docs + ordinal (bm25x_search_batch_growing): the sum obeys check_common's
    // bound on n_docs, so that every merged id stays below the BM25X_DOC_INF sentinel
    if ((uint64_t)NS + first + G > (uint64_t)BM25X_DOC_INF - 1u) {
        bm25x_set_error("%s: sealed n_docs=%u + growing n_docs=%llu exceeds %u documents (doc ids are 32-bit, %u is reserved)",
                        who, NS, (unsigned long long)first + G, BM25X_DOC_INF - 1u, BM25X_DOC_INF);
        return BM25X_ERR_INVALID;
    }
    // a batch with many postings against the vocabulary is grouped by counting over every term (O(T + P)), a small one by
    // a sort of its own postings (O(P log P)), so that an insert of one document costs no O(T) pass
    const uint64_t E = g->elem_off[G] >= g->elem_off[0] ? g->elem_off[G] - g->elem_off[0] : 0;
    const bool dense = E * 8 >= T;
    std::vector<uint64_t> cnt(dense ? (size_t)T + 1 : 0, 0);
    // pass 1: validate the documents and count their live postings (per term when dense)
    uint64_t P = 0;
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
            if (t >= T || sdf[t] == 0) continue;
            if (f >= (1u << 24)) bad |= 2;
            P++;
            if (dense) cnt[(size_t)t + 1]++;
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
    // pass 2: invert.  Documents are visited in ascending ordinal and grouped stably, so every list comes out ascending.
    auto live = [&](uint32_t d, uint64_t e) {
        const uint32_t t = g->elem_term[e];
        return !(g->deleted && g->deleted[d]) && t != BM25X_TERM_MISSING && t < T && sdf[t] != 0;
    };
    out = GrowingCsr();
    out.doc.resize(P);
    out.tf.resize(P);
    if (dense) {
        for (uint32_t t = 0; t < T; t++) cnt[(size_t)t + 1] += cnt[t];
        std::vector<uint64_t> cur(cnt.begin(), cnt.end() - 1);
        for (uint32_t d = 0; d < G; d++)
            for (uint64_t e = g->elem_off[d]; e < g->elem_off[d + 1]; e++)
                if (live(d, e)) {
                    const uint64_t p = cur[g->elem_term[e]]++;
                    out.doc[p] = first + d;
                    out.tf[p] = g->elem_tf[e];
                }
        for (uint32_t t = 0; t < T; t++)
            if (cnt[(size_t)t + 1] > cnt[t]) {
                out.term.push_back(t);
                out.off.push_back(cnt[(size_t)t + 1]);
            }
        return BM25X_OK;
    }
    std::vector<uint64_t> src;  // element index of each live posting, in document order
    src.reserve(P);
    for (uint32_t d = 0; d < G; d++)
        for (uint64_t e = g->elem_off[d]; e < g->elem_off[d + 1]; e++)
            if (live(d, e)) src.push_back(e);
    std::vector<uint32_t> owner(P);
    for (uint32_t d = 0, p = 0; d < G; d++)
        for (uint64_t e = g->elem_off[d]; e < g->elem_off[d + 1]; e++)
            if (live(d, e)) owner[p++] = first + d;
    std::vector<uint32_t> perm(P);
    for (uint32_t p = 0; p < P; p++) perm[p] = p;
    std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return g->elem_term[src[a]] < g->elem_term[src[b]]; });
    for (uint64_t i = 0; i < P; i++) {
        const uint32_t t = g->elem_term[src[perm[i]]];
        if (out.term.empty() || out.term.back() != t) {
            if (!out.term.empty()) out.off.push_back(i);
            out.term.push_back(t);
        }
        out.doc[i] = owner[perm[i]];
        out.tf[i] = g->elem_tf[src[perm[i]]];
    }
    if (!out.term.empty()) out.off.push_back(P);
    return BM25X_OK;
}

// Options of a growing segment's handle: the sealed side's `prune`, over the environment overrides handle_open applied,
// so that its searches take the sealed handles' kernel paths.
static void growing_options(bm25x_index *ix, const SealedSide &sealed) { ix->prune = sealed.home().prune; }

extern "C" int bm25x_growing_create(const bm25x_index *sealed, const bm25x_growing_docs *g, bm25x_index **out) {
    const char *who = "bm25x_growing_create";
    if (!sealed || !g || !out) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    const uint32_t G = g->n_docs, T = sealed->d.n_terms;
    SealedSide side;
    side.ix = const_cast<bm25x_index *>(sealed);  // read only
    GrowingCsr csr;
    int rc = invert_growing(side, g, 0, csr);
    if (rc != BM25X_OK) return rc;
    std::vector<uint32_t> df(T, 0);
    std::vector<uint64_t> off((size_t)T + 1, 0);
    for (size_t i = 0; i < csr.term.size(); i++) df[csr.term[i]] = (uint32_t)(csr.off[i + 1] - csr.off[i]);
    for (uint32_t t = 0; t < T; t++) off[(size_t)t + 1] = off[t] + df[t];
    const uint64_t P = off[T];
    BuildMeta m{G, T, g->doc_len, g->payload, sealed->h_keys.empty() ? nullptr : sealed->h_keys.data(), sealed->k1,
                sealed->b, df.data(), P};
    m.fieldnorm = g->doc_fieldnorm;
    const Stats st = side.stats();
    IndexGuard ix;
    rc = index_begin(m, &st, sealed->device, ix);
    if (rc == BM25X_OK) rc = upload_csr(ix.get(), who, T, P, off.data(), csr.doc.data(), csr.tf.data());
    if (rc != BM25X_OK) return rc;
    growing_options(ix.get(), side);
    *out = ix.release();
    return BM25X_OK;
}

// A 16-byte term key as two words, the key of the segment's key dictionary.
struct Key16 {
    uint64_t a, b;
    bool operator==(const Key16 &o) const { return a == o.a && b == o.b; }
};
struct Key16Hash {
    size_t operator()(const Key16 &k) const {
        const uint64_t h = (k.a ^ (k.b * 0x9E3779B97F4A7C15ull)) * 0xBF58476D1CE4E5B9ull;
        return (size_t)(h ^ (h >> 31));
    }
};
static Key16 key16(const uint8_t *p) {
    Key16 k;
    memcpy(&k.a, p, 8);
    memcpy(&k.b, p + 8, 8);
    return k;
}

// What a segment is bound to: its sealed side, the statistics it scores with (the sealed segment's, computed once) and,
// over a document-sharded side, that side's vocabulary on the home device (an index keeps its own,
// bm25x_index.key_vocab).  A call that reads the sealed side outside the segment's lock takes the binding under it,
// together with the handle, and holds its reference until it returns; a rebind swaps both in one step, then waits until
// the last holder of the old binding has dropped it (`released`, set by the rebind, fires in the destructor).
struct Binding {
    SealedSide sealed;
    Stats stats;
    int device;
    std::mutex vocab_mu;
    void *key_vocab = nullptr;
    std::promise<void> *released = nullptr;

    explicit Binding(const SealedSide &s) : sealed(s), stats(s.stats()), device(s.home().device) {}
    ~Binding() {
        if (key_vocab) {
            cudaSetDevice(device);
            cudaFree(key_vocab);
        }
        if (released) released->set_value();
    }
    // the vocabulary tsvector_rows casts against
    TsvVocab vocab() {
        if (sealed.ix) return {sealed.ix->device, &sealed.ix->h_keys, sealed.ix->d.n_terms, &sealed.ix->key_vocab,
                               &sealed.ix->key_vocab_mutex};
        return {device, &sealed.keys(), sealed.n_terms(), &key_vocab, &vocab_mu};
    }
};

// The record of a segment's latest successful seal, what its rebind needs (serial == 0: none): the serial of the handle
// it returned, its n_growing, growing map and term map.
struct SealRecord {
    uint64_t serial = 0;
    uint32_t n_growing = 0;
    std::vector<uint32_t> gmap, tmap;
};

// ---- the mutable growing segment (DESIGN §4.5): the documents on the host as the reference's VectorTuples keep them
// (norm, payload, deleted bit), their postings in one index handle on the sealed side's home device, brought up to date
// by a refresh ----
struct bm25x_growing_segment {
    const bool sharded;                // opened over a document-sharded index (a rebind keeps the kind)
    mutable std::mutex mu;             // guards everything below; a refresh runs under it
    // the binding (changed by a rebind only, under mu and num_mu)
    std::shared_ptr<Binding> bind;
    SealRecord last_seal;
    int norm_form = -1;                // -1: no insert yet; 1: doc_len; 0: doc_fieldnorm
    std::vector<uint8_t> fieldnorm;    // per ordinal
    std::vector<uint32_t> doc_len;     // per ordinal (doc_len form only)
    std::vector<uint16_t> payload;     // per ordinal x 3: the given ctid, or the synthetic one of the ordinal
    std::vector<uint8_t> deleted;      // per ordinal
    uint32_t n_deleted = 0;
    // postings inserted since the last refresh, one entry per posting: each insert's term-major CSR appended as it came,
    // so that the postings of one term are in insertion order, hence ordinals ascending
    std::vector<uint32_t> pend_term, pend_doc, pend_tf;
    bool pending = false;              // inserts or deletes since the last refresh
    // what only the seal reads (bm25x_growing_seal): the "dormant" postings the handle never holds (terms >= the sealed
    // n_terms, terms without sealed postings) of every document not inserted deleted, as (term, ordinal, tf) appended per
    // insert; in doc_fieldnorm form each ordinal's saturating Σ tf over all its elements (Document::length,
    // vector.rs:77-83); the inserted ordinals >= the sealed n_terms, each once, in the order they first came
    std::vector<uint32_t> dorm_term, dorm_doc, dorm_tf;
    std::vector<uint32_t> sum_tf;
    std::vector<uint32_t> new_terms;
    std::unordered_set<uint32_t> new_seen;
    uint32_t term_end = 0;             // 1 + the largest ordinal in new_terms (0: none)
    // the current handle over ordinals [0, n_indexed); a running search keeps its own reference, so that a refresh can
    // replace it meanwhile and the last holder destroys it
    std::shared_ptr<bm25x_index> cur;
    // the keys the segment numbered (bm25x_growing_insert_tsvectors): key i has ordinal n_terms(sealed) + i.  The segment
    // owns its keys from its first tsvector insert on.  num_mu is held across a whole tsvector insert, so that keys are
    // numbered in commit order; the keys change under both locks.
    std::mutex num_mu;
    bool owns_keys = false;
    std::vector<uint8_t> new_keys;
    std::unordered_map<Key16, uint32_t, Key16Hash> key_ord;

    explicit bm25x_growing_segment(const SealedSide &s) : sharded(s.sx != nullptr), bind(std::make_shared<Binding>(s)) {}
    uint32_t n_docs() const { return (uint32_t)deleted.size(); }
    uint32_t n_keys() const { return (uint32_t)(new_keys.size() / 16); }
    // the sealed side, under mu or num_mu
    const SealedSide &sealed() const { return bind->sealed; }
    // the binding, for a call that reads it outside the lock
    std::shared_ptr<Binding> binding() const {
        std::lock_guard<std::mutex> lock(mu);
        return bind;
    }
};

extern "C" int bm25x_growing_open(bm25x_index *sealed, bm25x_growing_segment **out) {
    if (!sealed || !out) {
        bm25x_set_error("bm25x_growing_open: null argument");
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    if (sealed->h_df.size() != sealed->d.n_terms) {
        bm25x_set_error("bm25x_growing_open: replica not finalized (bm25x_index_finalize_replica)");
        return BM25X_ERR_INVALID;
    }
    SealedSide side;
    side.ix = sealed;
    *out = new bm25x_growing_segment(side);
    return BM25X_OK;
}

extern "C" int bm25x_growing_open_sharded(bm25x_sharded_index *sealed, bm25x_growing_segment **out) {
    if (!sealed || !out) {
        bm25x_set_error("bm25x_growing_open_sharded: null argument");
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    SealedSide side;
    side.sx = sealed;
    *out = new bm25x_growing_segment(side);
    return BM25X_OK;
}

extern "C" void bm25x_growing_close(bm25x_growing_segment *g) { delete g; }

// bm25x_growing_insert under g->mu.  sealed_only: every ordinal must be a sealed one or BM25X_TERM_MISSING (the segment
// owns its keys).
static int growing_insert_locked(bm25x_growing_segment *g, const bm25x_growing_docs *docs, bool sealed_only) {
    const int form = docs->doc_len ? 1 : docs->doc_fieldnorm ? 0 : -1;
    if (g->norm_form >= 0 && form >= 0 && form != g->norm_form) {
        bm25x_set_error("bm25x_growing_insert: documents with %s into a segment whose documents carry %s",
                        form ? "doc_len" : "doc_fieldnorm", form ? "doc_fieldnorm" : "doc_len");
        return BM25X_ERR_INVALID;
    }
    const uint32_t first = g->n_docs(), G = docs->n_docs;
    GrowingCsr csr;
    const int rc = invert_growing(g->sealed(), docs, first, csr);
    if (rc != BM25X_OK) return rc;
    for (uint32_t d = 0; sealed_only && d < G; d++)  // (invert_growing checked the offsets)
        for (uint64_t e = docs->elem_off[d]; e < docs->elem_off[d + 1]; e++) {
            const uint32_t t = docs->elem_term[e];
            if (t >= g->sealed().n_terms() && t != BM25X_TERM_MISSING) {
                bm25x_set_error("bm25x_growing_insert: document %u holds term ordinal %u >= n_terms(sealed)=%u, but the "
                                "segment numbers its new terms itself (bm25x_growing_insert_tsvectors)", d, t,
                                g->sealed().n_terms());
                return BM25X_ERR_INVALID;
            }
        }
    g->norm_form = form;
    g->fieldnorm.resize((size_t)first + G);
    if (form) {
        g->doc_len.insert(g->doc_len.end(), docs->doc_len, docs->doc_len + G);
        for (uint32_t d = 0; d < G; d++) g->fieldnorm[(size_t)first + d] = bm25x_length_to_fieldnorm(docs->doc_len[d]);
    } else {
        std::copy(docs->doc_fieldnorm, docs->doc_fieldnorm + G, g->fieldnorm.begin() + first);
    }
    g->payload.resize(((size_t)first + G) * 3);
    for (uint32_t d = 0; d < G; d++) {
        uint16_t *p = &g->payload[((size_t)first + d) * 3];
        if (docs->payload) std::copy(docs->payload + (size_t)d * 3, docs->payload + (size_t)d * 3 + 3, p);
        else synth_ctid(first + d, p);
    }
    g->deleted.resize((size_t)first + G, 0);
    for (uint32_t d = 0; docs->deleted && d < G; d++)
        if (docs->deleted[d]) {
            g->deleted[(size_t)first + d] = 1;
            g->n_deleted++;
        }
    for (size_t i = 0; i < csr.term.size(); i++)
        g->pend_term.insert(g->pend_term.end(), csr.off[i + 1] - csr.off[i], csr.term[i]);
    g->pend_doc.insert(g->pend_doc.end(), csr.doc.begin(), csr.doc.end());
    g->pend_tf.insert(g->pend_tf.end(), csr.tf.begin(), csr.tf.end());
    // the seal's share: dormant postings, Σ tf (doc_fieldnorm form), new ordinals
    const uint32_t T = g->sealed().n_terms();
    const std::vector<uint32_t> &sdf = g->sealed().df();
    for (uint32_t d = 0; d < G; d++) {
        const bool live = !(docs->deleted && docs->deleted[d]);
        uint64_t sum = 0;
        for (uint64_t e = docs->elem_off[d]; e < docs->elem_off[d + 1]; e++) {
            const uint32_t t = docs->elem_term[e];
            sum += docs->elem_tf[e];
            if (t == BM25X_TERM_MISSING) continue;
            if (t >= T && g->new_seen.insert(t).second) {
                g->new_terms.push_back(t);
                g->term_end = std::max(g->term_end, t + 1);
            }
            if (live && (t >= T || sdf[t] == 0)) {
                g->dorm_term.push_back(t);
                g->dorm_doc.push_back(first + d);
                g->dorm_tf.push_back(docs->elem_tf[e]);
            }
        }
        if (!form) g->sum_tf.push_back((uint32_t)std::min<uint64_t>(sum, 0xFFFFFFFFu));
    }
    g->pending = true;
    return BM25X_OK;
}

extern "C" int bm25x_growing_insert(bm25x_growing_segment *g, const bm25x_growing_docs *docs) {
    if (!g || !docs) {
        bm25x_set_error("bm25x_growing_insert: null argument");
        return BM25X_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(g->mu);
    return growing_insert_locked(g, docs, g->owns_keys);
}

// A segment that took ordinals >= n_terms(sealed) from bm25x_growing_insert cannot number keys itself (under g->mu).
static int check_caller_numbered(const char *who, const bm25x_growing_segment *g) {
    if (g->owns_keys || g->new_terms.empty()) return BM25X_OK;
    bm25x_set_error("%s: the segment holds term ordinal %u >= n_terms(sealed)=%u from bm25x_growing_insert: its new terms "
                    "are numbered by the caller", who, g->new_terms[0], g->sealed().n_terms());
    return BM25X_ERR_INVALID;
}

// A sealed side without term keys: bm25x_lookup_terms' refusal (bm25x_sharded_lookup_terms gives the same).
static int check_keyed(const SealedSide &s) {
    if (!s.keys().empty() || !s.n_terms()) return BM25X_OK;
    bm25x_set_error("bm25x_lookup_terms: index was created without term keys");
    return BM25X_ERR_INVALID;
}

extern "C" int bm25x_growing_insert_tsvectors(bm25x_growing_segment *g, const uint8_t seed[32], const bm25x_tsvectors *tsv,
                                              const uint16_t *payload) {
    const char *who = "bm25x_growing_insert_tsvectors";
    if (!g || !seed || !tsv) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_tsvectors(who, tsv, 0);
    if (rc != BM25X_OK) return rc;
    // num_mu also holds the binding: only a rebind changes it, and a rebind takes num_mu first
    std::lock_guard<std::mutex> numbering(g->num_mu);
    rc = check_keyed(g->sealed());
    if (rc != BM25X_OK) return rc;
    {
        std::lock_guard<std::mutex> lock(g->mu);
        rc = check_caller_numbered(who, g);
        if (rc != BM25X_OK) return rc;
    }
    // the call's keys the sealed vocabulary lacks: the ordinal an earlier insert gave, or the next fresh one in key order
    // (g->key_ord changes only under num_mu, held here)
    const uint32_t T = g->sealed().n_terms(), K = g->n_keys();
    std::vector<uint8_t> fresh;
    auto number = [&](uint32_t nu, const uint8_t *keys, uint32_t *ord) {
        for (uint32_t i = 0; i < nu; i++) {
            const auto it = g->key_ord.find(key16(keys + (size_t)i * 16));
            if (it != g->key_ord.end()) {
                ord[i] = it->second;
                continue;
            }
            const uint64_t t = (uint64_t)T + K + fresh.size() / 16;
            if (t >= BM25X_TERM_MISSING) {
                bm25x_set_error("%s: more than %u term ordinals (%u is BM25X_TERM_MISSING)", who, BM25X_TERM_MISSING,
                                BM25X_TERM_MISSING);
                return BM25X_ERR_UNSUPPORTED;
            }
            ord[i] = (uint32_t)t;
            fresh.insert(fresh.end(), keys + (size_t)i * 16, keys + (size_t)i * 16 + 16);
        }
        return BM25X_OK;
    };
    TsvRows r;
    rc = tsvector_rows(who, g->bind->vocab(), seed, tsv, 0, number, r);
    if (rc != BM25X_OK) return rc;
    // the restated rows go in as bm25x_growing_insert takes them, with the norm in the segment's form
    bm25x_growing_docs d{};
    d.n_docs = tsv->n;
    d.payload = payload;
    d.elem_off = r.off.data();
    d.elem_term = r.ord.data();
    d.elem_tf = r.tf.data();
    std::lock_guard<std::mutex> lock(g->mu);
    std::vector<uint8_t> fn;
    if (g->norm_form == 0) {
        fn.resize(r.len.size());
        for (size_t i = 0; i < fn.size(); i++) fn[i] = bm25x_length_to_fieldnorm(r.len[i]);
        d.doc_fieldnorm = fn.data();
    } else {
        d.doc_len = r.len.data();
    }
    rc = check_caller_numbered(who, g);  // an ordinal insert may have come meanwhile
    if (rc == BM25X_OK) rc = growing_insert_locked(g, &d, false);
    if (rc != BM25X_OK) return rc;
    for (size_t i = 0; i < fresh.size() / 16; i++) g->key_ord.emplace(key16(&fresh[i * 16]), (uint32_t)(T + K + i));
    g->new_keys.insert(g->new_keys.end(), fresh.begin(), fresh.end());
    g->owns_keys = true;
    return BM25X_OK;
}

extern "C" int bm25x_growing_get_new_keys(const bm25x_growing_segment *g, uint32_t cap, uint8_t *keys_out, uint32_t *n_out) {
    const char *who = "bm25x_growing_get_new_keys";
    if (!g || !n_out || (cap && !keys_out)) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(g->mu);
    const uint32_t K = g->n_keys();
    *n_out = K;
    if (cap < K) {
        bm25x_set_error("%s: cap=%u below the segment's %u keys", who, cap, K);
        return BM25X_ERR_INVALID;
    }
    if (K) memcpy(keys_out, g->new_keys.data(), g->new_keys.size());
    return BM25X_OK;
}

extern "C" int bm25x_growing_tsvector_queries(bm25x_growing_segment *g, const uint8_t seed[32], const bm25x_tsvectors *tsv,
                                              uint32_t *q_off, uint32_t *q_terms) {
    const char *who = "bm25x_growing_tsvector_queries";
    if (!g || !seed || !tsv || !q_off) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    int rc = check_tsvectors(who, tsv, 1);
    if (rc != BM25X_OK) return rc;
    if (!q_terms && tsv->ent_off[tsv->n]) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    const std::shared_ptr<Binding> bind = g->binding();
    rc = check_keyed(bind->sealed);
    if (rc != BM25X_OK) return rc;
    // keys the segment numbered are not in the sealed vocabulary: BM25X_TERM_MISSING, as before the seal they never match
    TsvRows r;
    rc = tsvector_rows(who, bind->vocab(), seed, tsv, 1, {}, r);
    if (rc != BM25X_OK) return rc;
    const uint64_t E = r.off[tsv->n];
    if (E > 0xFFFFFFFFull) {
        bm25x_set_error("%s: %llu query terms, more than the 2^32 - 1 that u32 offsets address", who, (unsigned long long)E);
        return BM25X_ERR_UNSUPPORTED;
    }
    if (E) memcpy(q_terms, r.ord.data(), sizeof(uint32_t) * E);
    for (uint32_t v = 0; v <= tsv->n; v++) q_off[v] = (uint32_t)r.off[v];
    return BM25X_OK;
}

extern "C" int bm25x_growing_delete(bm25x_growing_segment *g, uint32_t n, const uint32_t *ordinals) {
    if (!g || (n && !ordinals)) {
        bm25x_set_error("bm25x_growing_delete: null argument");
        return BM25X_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(g->mu);
    const uint32_t N = g->n_docs();
    for (uint32_t i = 0; i < n; i++)
        if (ordinals[i] >= N) {
            bm25x_set_error("bm25x_growing_delete: ordinal %u (entry %u) >= n_docs=%u", ordinals[i], i, N);
            return BM25X_ERR_INVALID;
        }
    for (uint32_t i = 0; i < n; i++)
        if (!g->deleted[ordinals[i]]) {
            g->deleted[ordinals[i]] = 1;
            g->n_deleted++;
            g->pending = true;
        }
    return BM25X_OK;
}

// ---- the splice of the refresh and the seal (bm25x_splice.cuh): the sources described, their survivors counted per
// term, a handle opened with that df, the survivors written into it ----

// The grid of a one-warp-per-term launch over n > 0 terms: 8 warps per block, at most 32 blocks per SM.
static unsigned splice_grid(uint32_t n, int sm_count) {
    return (unsigned)std::min<uint64_t>(((uint64_t)n + 7) / 8, (uint64_t)sm_count * 32ull);
}

// The deleted bitmap of a byte-per-document vector: bit d of word d >> 5 set = deleted[d] != 0.
static std::vector<uint32_t> deleted_bitmap(const std::vector<uint8_t> &deleted) {
    std::vector<uint32_t> bits((deleted.size() + 31) / 32, 0);
    for (size_t d = 0; d < deleted.size(); d++)
        if (deleted[d]) bits[d >> 5] |= 1u << (d & 31);
    return bits;
}

// An index handle's lists as a splice source (h == NULL: no source).
static SpliceSrc handle_source(const bm25x_index *h, const uint32_t *del, const uint32_t *map) {
    SpliceSrc s{};
    if (h) {
        s.off = h->d.post_off;
        s.df = h->d.df;
        s.doc = h->d.pdoc;
        s.post = h->d.post;
        s.n_terms = h->d.n_terms;
    }
    s.del = del;
    s.map = map;
    return s;
}

// A (term, doc, tf) list, appended so that each term's docs ascend, grouped over n terms and uploaded as a splice source:
// a stable counting sort by term keeps each term's docs in order.  Failures stick in sc.e.
static SpliceSrc grouped_source(Scratch &sc, uint32_t n, const std::vector<uint32_t> &term, const std::vector<uint32_t> &doc,
                                const std::vector<uint32_t> &tf, const uint32_t *del, const uint32_t *map) {
    const uint64_t P = term.size();
    std::vector<uint64_t> off((size_t)n + 1, 0);
    for (uint64_t p = 0; p < P; p++) off[(size_t)term[p] + 1]++;
    for (uint32_t t = 0; t < n; t++) off[(size_t)t + 1] += off[t];
    std::vector<uint32_t> gdoc(P), gtf(P);
    std::vector<uint64_t> at(off.begin(), off.end() - 1);
    for (uint64_t p = 0; p < P; p++) {
        const uint64_t i = at[term[p]]++;
        gdoc[i] = doc[p];
        gtf[i] = tf[p];
    }
    SpliceSrc s{};
    s.off = sc.up(off.data(), off.size());
    s.doc = sc.up(gdoc.data(), P);
    s.tf = sc.up(gtf.data(), P);
    s.del = del;
    s.map = map;
    s.n_terms = n;
    return s;
}

// df[t] = the surviving postings of term t < n over src: k_splice_count, then the download.  Failures stick in sc.e.
static std::vector<uint32_t> splice_count(Scratch &sc, int sm_count, uint32_t n, const SpliceSources &src) {
    std::vector<uint32_t> df(n);
    uint32_t *d_df = sc.alloc<uint32_t>(n);
    if (sc.e == cudaSuccess && n) {
        k_splice_count<<<splice_grid(n, sm_count), 256>>>(n, src, d_df);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess && n) sc.e = cudaMemcpy(df.data(), d_df, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost);
    return df;
}

// The survivors of src written into ix, opened by index_begin with the df splice_count gave (new term j from source term
// src_of[j]; src_of == NULL: j), then what every index derives from them.  A CUDA failure, here or earlier in sc.e, is
// refused as step "splice" of `who`.
static int splice_finish(Scratch &sc, const char *who, bm25x_index *ix, const uint32_t *src_of, const SpliceSources &src) {
    const uint32_t n = ix->d.n_terms;
    if (sc.e == cudaSuccess && n) {
        k_splice<<<splice_grid(n, ix->sm_count), 256>>>(n, src_of, src, ix->d.fieldnorm, ix->d.post_off, ix->d.post);
        sc.e = cudaGetLastError();
    }
    if (sc.e == cudaSuccess) sc.e = cudaDeviceSynchronize();
    if (sc.e == cudaSuccess) sc.e = index_finish_device(ix);
    return sc.e == cudaSuccess ? BM25X_OK : cuda_refusal(who, "splice", sc.e);
}

// The refresh, under g->mu: the next handle is built beside the current one (which running searches may still read)
// from its surviving postings and the inserted ones, then replaces it.  On a refusal nothing changes.
static int growing_refresh_locked(bm25x_growing_segment *g) {
    const char *who = "bm25x_growing_refresh";
    if (!g->pending) return BM25X_OK;
    const bm25x_index &home = g->sealed().home();
    const std::vector<uint8_t> &keys = g->sealed().keys();
    const uint32_t N = g->n_docs(), T = g->sealed().n_terms();
    const int device = home.device;
    // ---- the sources: the current handle's lists, then the postings inserted since, against the deleted ordinals ----
    Scratch sc(device);
    sc.e = cudaSetDevice(device);
    const std::vector<uint32_t> bits = deleted_bitmap(g->deleted);
    const uint32_t *d_del = sc.up(bits.data(), bits.size());
    SpliceSources src{};
    src.s[0] = handle_source(g->cur.get(), d_del, nullptr);
    src.s[1] = grouped_source(sc, T, g->pend_term, g->pend_doc, g->pend_tf, d_del, nullptr);
    // ---- new df: the survivors of the current lists and of the inserted ones ----
    const std::vector<uint32_t> df = splice_count(sc, home.sm_count, T, src);
    if (sc.e != cudaSuccess) return cuda_refusal(who, "count", sc.e);
    uint64_t P = 0;
    for (uint32_t t = 0; t < T; t++) P += df[t];
    // ---- the new handle, built as bm25x_growing_create builds one over all N ordinals ----
    BuildMeta m{N, T, g->norm_form ? g->doc_len.data() : nullptr, g->payload.data(), keys.empty() ? nullptr : keys.data(),
                home.k1, home.b, df.data(), P};
    m.fieldnorm = g->norm_form ? nullptr : g->fieldnorm.data();
    IndexGuard ix;
    int rc = index_begin(m, &g->bind->stats, device, ix);
    if (rc == BM25X_OK) rc = splice_finish(sc, who, ix.get(), nullptr, src);
    if (rc != BM25X_OK) return rc;
    growing_options(ix.get(), g->sealed());
    g->cur.reset(ix.release(), IndexDestroy());
    std::vector<uint32_t>().swap(g->pend_term);
    std::vector<uint32_t>().swap(g->pend_doc);
    std::vector<uint32_t>().swap(g->pend_tf);
    g->pending = false;
    return BM25X_OK;
}

extern "C" int bm25x_growing_refresh(bm25x_growing_segment *g) {
    if (!g) {
        bm25x_set_error("bm25x_growing_refresh: null argument");
        return BM25X_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(g->mu);
    return growing_refresh_locked(g);
}

extern "C" int bm25x_growing_get_info(const bm25x_growing_segment *g, bm25x_growing_info *out) {
    if (!g || !out) {
        bm25x_set_error("bm25x_growing_get_info: null argument");
        return BM25X_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(g->mu);
    memset(out, 0, sizeof(*out));
    out->n_docs = g->n_docs();
    out->n_deleted = g->n_deleted;
    out->n_postings = g->cur ? g->cur->d.n_post : 0;
    out->device_bytes = g->cur ? g->cur->device_bytes : 0;
    out->pending = g->pending ? 1u : 0u;
    out->device = g->sealed().home().device;
    return BM25X_OK;
}

extern "C" int bm25x_growing_get_index(const bm25x_growing_segment *g, bm25x_index_layout *layout,
                                       bm25x_index_derived *derived) {
    if (!g) {
        bm25x_set_error("bm25x_growing_get_index: null argument");
        return BM25X_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lock(g->mu);
    if (!g->cur) {
        bm25x_set_error("bm25x_growing_get_index: no document has been indexed yet (insert, then refresh)");
        return BM25X_ERR_INVALID;
    }
    int rc = layout ? bm25x_index_get_layout(g->cur.get(), layout) : BM25X_OK;
    if (rc == BM25X_OK && derived) rc = bm25x_index_get_derived(g->cur.get(), derived);
    return rc;
}

extern "C" int bm25x_growing_search_batch(bm25x_growing_segment *g, uint32_t nq, const uint32_t *q_off,
                                          const uint32_t *q_terms, uint32_t k, const uint8_t *allow_sealed,
                                          const uint8_t *allow_growing, uint32_t allow_growing_docs, uint32_t *out_doc,
                                          float *out_score, double *out_score64, uint16_t *out_payload, uint32_t *out_n,
                                          bm25x_search_stats *stats) {
    if (!g) {
        bm25x_set_error("bm25x_growing_search_batch: null argument");
        return BM25X_ERR_INVALID;
    }
    if (const int rc = check_k(k, false); rc != BM25X_OK) return rc;  // before the refresh: a refused call leaves it pending
    const auto t0 = std::chrono::steady_clock::now();
    // this search's state of the segment: its binding and its handle (NULL: nothing inserted yet), taken as one
    std::shared_ptr<Binding> bind;
    std::shared_ptr<bm25x_index> cur;
    {
        std::lock_guard<std::mutex> lock(g->mu);
        const int rc = growing_refresh_locked(g);
        if (rc != BM25X_OK) return rc;
        bind = g->bind;
        cur = g->cur;
    }
    std::vector<uint8_t> ag;  // allow_growing over the handle's ordinals: the caller's bits below allow_growing_docs
    if (cur && allow_growing) {
        const uint32_t N = cur->d.n_docs, n = std::min(N, allow_growing_docs);
        ag.assign(((size_t)N + 7) / 8, 0);
        std::copy(allow_growing, allow_growing + ((size_t)n + 7) / 8, ag.begin());
        if (n & 7u) ag[n >> 3] &= (uint8_t)((1u << (n & 7u)) - 1u);
    }
    SideFilter f;
    f.allow_sealed = allow_sealed;
    f.allow_growing = cur && allow_growing ? ag.data() : nullptr;
    return sealed_side_search("bm25x_growing_search_batch", bind->sealed, cur.get(), f, true, nq, q_off, q_terms, k,
                              {out_doc, out_score, out_score64, out_payload, out_n}, stats, t0);
}

extern "C" int bm25x_growing_search_candidates(bm25x_growing_segment *g, uint32_t nq, const uint32_t *q_off,
                                               const uint32_t *q_terms, const uint32_t *c_off, const uint32_t *c_docs,
                                               uint32_t k, uint32_t *out_doc, float *out_score, double *out_score64,
                                               uint16_t *out_payload, uint32_t *out_n, bm25x_search_stats *stats) {
    const char *who = "bm25x_growing_search_candidates";
    if (!g || (nq && (!c_off || (!c_docs && c_off[nq] != 0)))) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    if (const int rc = check_k(k, false); rc != BM25X_OK) return rc;  // before the refresh: a refused call leaves it pending
    const auto t0 = std::chrono::steady_clock::now();
    std::shared_ptr<Binding> bind;
    std::shared_ptr<bm25x_index> cur;
    {
        std::lock_guard<std::mutex> lock(g->mu);
        const int rc = growing_refresh_locked(g);
        if (rc != BM25X_OK) return rc;
        bind = g->bind;
        cur = g->cur;
    }
    // before the first insert the sealed side alone answers: its ids are the only ones
    if (!cur)
        if (const int rc = check_candidates(who, nq, c_off, c_docs, bind->sealed.n_docs()); rc != BM25X_OK) return rc;
    SideFilter f;
    f.c_off = c_off;
    f.c_docs = c_docs;
    return sealed_side_search(who, bind->sealed, cur.get(), f, true, nq, q_off, q_terms, k,
                              {out_doc, out_score, out_score64, out_payload, out_n}, stats, t0);
}

// ---- the seal (`maintain`, maintain.rs:27-311; DESIGN §4.5): a new sealed index from the sealed survivors and the
// segment's, built on the device from the arrays already there ----

// What the seal reads of the segment, copied under its lock right after a refresh.
struct SealSnapshot {
    uint32_t n = 0;                    // ordinals
    std::shared_ptr<bm25x_index> cur;  // the refreshed handle over them (NULL: none)
    std::vector<uint8_t> deleted;
    std::vector<uint32_t> len;         // rule 4 length per ordinal: doc_len, or Σ tf in doc_fieldnorm form
    std::vector<uint16_t> payload;
    std::vector<uint32_t> dorm_term, dorm_doc, dorm_tf;
};

// The seal of g over its sealed side's parts (one index: one part; a document-sharded index: its shards).  New part j
// holds the survivors of an old part in ascending old id, the last one also the growing survivors after its own; a part
// left without a document is dropped.  Each part is counted and spliced on its own device from its own arrays; the host
// sums df over the parts, settles the vocabulary and builds ONE Stats for the new segment, with which every new handle
// is opened.  The new segment is handed out in *out as a document-sharded index, one shard per part that keeps a document;
// until then bm25x_sharded_destroy holds it, so that a refusal frees every handle built so far.  Refusals and maps are
// bm25x_growing_seal's, named by `who`.
static int seal_segment(const char *who, bm25x_growing_segment *g, bm25x_seal_args *a, bm25x_sharded_index **out) {
    const std::shared_ptr<Binding> bind = g->binding();  // held to the end: a rebind waits for it
    const SealedSide &sealed = bind->sealed;
    const uint32_t NS = sealed.n_docs(), T = sealed.n_terms();
    uint32_t K = a->n_new_keys;
    bool keyed = !sealed.keys().empty();
    // ---- the new keys: each unlike every sealed key and every other new key.  The caller's, or (taken with the
    // snapshot below) those the segment owns, which are so by construction ----
    if (a->new_keys && !keyed) {
        bm25x_set_error("%s: new_keys given, but the sealed index was created without term keys", who);
        return BM25X_ERR_INVALID;
    }
    const uint8_t *skeys = sealed.keys().data(), *nkeys = a->new_keys;
    std::vector<uint8_t> owned;
    auto key_of = [&](uint32_t t) { return t < T ? skeys + (size_t)t * 16 : nkeys + (size_t)(t - T) * 16; };
    auto key_less = [&](uint32_t x, uint32_t y) { return memcmp(key_of(x), key_of(y), 16) < 0; };
    if (K) {
        std::vector<uint32_t> order(K);
        for (uint32_t i = 0; i < K; i++) order[i] = T + i;
        std::sort(order.begin(), order.end(), key_less);
        for (uint32_t i = 1; i < K; i++)
            if (memcmp(key_of(order[i - 1]), key_of(order[i]), 16) == 0) {
                const uint32_t x = std::min(order[i - 1], order[i]) - T, y = std::max(order[i - 1], order[i]) - T;
                bm25x_set_error("%s: new key %u equals new key %u", who, x, y);
                return BM25X_ERR_INVALID;
            }
        for (uint32_t i = 0; i < K; i++) {
            const uint32_t t = key_ordinal(skeys, T, key_of(T + i));
            if (t != BM25X_TERM_MISSING) {
                bm25x_set_error("%s: new key %u equals the key of sealed term %u", who, i, t);
                return BM25X_ERR_INVALID;
            }
        }
    }
    // ---- rule 1: the sealed survivors in ascending old id ----
    std::vector<uint32_t> smap(NS);
    uint32_t ns_keep = 0;
    for (uint32_t d = 0; d < NS; d++)
        smap[d] = a->sealed_deleted && ((a->sealed_deleted[d >> 3] >> (d & 7u)) & 1u) ? BM25X_DOC_INF : ns_keep++;
    // ---- the snapshot: every refusal that depends on the segment first, then a refresh and a copy ----
    SealSnapshot s;
    uint32_t n_src;
    {
        std::lock_guard<std::mutex> lock(g->mu);
        if (g->bind != bind) {
            bm25x_set_error("%s: the segment was rebound while the seal began: seal it again", who);
            return BM25X_ERR_INVALID;
        }
        const uint32_t NG = g->n_docs();
        if (g->owns_keys) {
            if (a->new_keys || a->n_new_keys) {
                bm25x_set_error("%s: new_keys given, but the segment numbered its new terms itself "
                                "(bm25x_growing_insert_tsvectors): it supplies their keys", who);
                return BM25X_ERR_INVALID;
            }
            owned = g->new_keys;
            nkeys = owned.data();
            K = g->n_keys();
            keyed = true;
        }
        n_src = keyed ? T + K : std::max(T, g->term_end);
        if (keyed)
            for (uint32_t t : g->new_terms)
                if (t >= T + K) {
                    bm25x_set_error("%s: inserted term ordinal %u >= n_terms(sealed)=%u + n_new_keys=%u (it has no key)", who,
                                    t, T, K);
                    return BM25X_ERR_INVALID;
                }
        if ((a->growing_map && NG > a->growing_cap) || (a->term_map && n_src > a->term_cap)) {
            a->n_growing = NG;
            a->n_source_terms = n_src;
            bm25x_set_error("%s: growing_cap=%u / term_cap=%u below n_growing=%u / n_source_terms=%u", who, a->growing_cap,
                            a->term_cap, NG, n_src);
            return BM25X_ERR_INVALID;
        }
        if (ns_keep == 0 && NG == g->n_deleted) {
            bm25x_set_error("%s: no document survives (every sealed and growing document is deleted)", who);
            return BM25X_ERR_INVALID;
        }
        for (size_t i = 0; i < g->dorm_tf.size(); i++)
            if (g->dorm_tf[i] >= (1u << 24) && !g->deleted[g->dorm_doc[i]]) {
                bm25x_set_error("%s: term frequency >= 2^24 is not supported by the packed posting layout", who);
                return BM25X_ERR_UNSUPPORTED;
            }
        const int rc = growing_refresh_locked(g);
        if (rc != BM25X_OK) return rc;
        s.n = NG;
        s.cur = g->cur;
        s.deleted = g->deleted;
        s.len = g->norm_form == 1 ? g->doc_len : g->sum_tf;
        s.payload = g->payload;
        s.dorm_term = g->dorm_term;
        s.dorm_doc = g->dorm_doc;
        s.dorm_tf = g->dorm_tf;
    }
    // ---- rule 1: the growing survivors after the sealed ones, in ascending ordinal ----
    const uint32_t NG = s.n;
    std::vector<uint32_t> gmap(NG);
    uint32_t N = ns_keep;
    for (uint32_t o = 0; o < NG; o++) gmap[o] = s.deleted[o] ? BM25X_DOC_INF : N++;
    // ---- per part: its survivors' new ids [new_lo, new_lo + n_new) (the last part's include the growing survivors) ----
    const std::vector<SealPart> parts = sealed.parts();
    const uint32_t NP = (uint32_t)parts.size();
    std::vector<uint32_t> new_lo(NP + 1, 0);
    for (uint32_t p = 0; p < NP; p++) {
        uint32_t kept = 0;
        for (uint32_t d = parts[p].first; d < parts[p].first + parts[p].n; d++) kept += smap[d] != BM25X_DOC_INF;
        new_lo[p + 1] = new_lo[p] + kept;
    }
    new_lo[NP] = N;
    // ---- per part, on its own device with its local ids: the sources (its sealed lists; the last part also the growing
    // handle's and the dormant postings), the local deleted bitmaps and maps, rule 3 lengths and rule 5 df ----
    const std::vector<uint32_t> gbits = deleted_bitmap(s.deleted);
    std::vector<std::unique_ptr<Scratch>> scs(NP);
    std::vector<SpliceSources> srcs(NP);
    std::vector<std::vector<uint32_t>> df_part(NP);
    std::vector<uint32_t> df_src(n_src, 0), len(N);
    std::vector<uint16_t> pay((size_t)N * 3);
    for (uint32_t p = 0; p < NP; p++) {
        const SealPart &pt = parts[p];
        const bool last = p + 1 == NP;
        Scratch &sc = *(scs[p] = std::make_unique<Scratch>(pt.h->device));
        sc.e = cudaSetDevice(pt.h->device);
        std::vector<uint32_t> sbits(((size_t)pt.n + 31) / 32, 0), lmap(pt.n);
        for (uint32_t d = 0; d < pt.n; d++) {
            const uint32_t nd = smap[pt.first + d];
            lmap[d] = nd == BM25X_DOC_INF ? nd : nd - new_lo[p];
            if (nd == BM25X_DOC_INF) sbits[d >> 5] |= 1u << (d & 31);
        }
        const uint32_t *d_sdel = sc.up(sbits.data(), sbits.size());
        SpliceSources &src = srcs[p];
        src = SpliceSources{};
        src.s[0] = handle_source(pt.h, d_sdel, sc.up(lmap.data(), pt.n));
        if (last) {
            std::vector<uint32_t> glmap(NG);
            for (uint32_t o = 0; o < NG; o++) glmap[o] = gmap[o] == BM25X_DOC_INF ? gmap[o] : gmap[o] - new_lo[p];
            const uint32_t *d_gdel = sc.up(gbits.data(), gbits.size()), *d_gmap = sc.up(glmap.data(), NG);
            src.s[1] = handle_source(s.cur.get(), d_gdel, d_gmap);
            src.s[2] = grouped_source(sc, n_src, s.dorm_term, s.dorm_doc, s.dorm_tf, d_gdel, d_gmap);
        }
        uint32_t *d_cnt = sc.alloc<uint32_t>(pt.n);
        const DeviceIndex &sd = pt.h->d;
        if (sc.e == cudaSuccess) sc.e = cudaMemset(d_cnt, 0, sizeof(uint32_t) * (size_t)pt.n);
        if (sc.e == cudaSuccess && T) {
            k_seal_doc_postings<<<splice_grid(T, pt.h->sm_count), 256>>>(T, sd.pdoc, sd.post_off, sd.df, d_sdel, d_cnt);
            sc.e = cudaGetLastError();
        }
        df_part[p] = splice_count(sc, pt.h->sm_count, n_src, src);
        std::vector<uint32_t> cnt(pt.n);
        std::vector<uint16_t> spay((size_t)pt.n * 3);
        if (sc.e == cudaSuccess) sc.e = cudaMemcpy(cnt.data(), d_cnt, sizeof(uint32_t) * (size_t)pt.n, cudaMemcpyDeviceToHost);
        if (sc.e == cudaSuccess)
            sc.e = cudaMemcpy(spay.data(), sd.payload, sizeof(uint16_t) * 3 * (size_t)pt.n, cudaMemcpyDeviceToHost);
        if (sc.e != cudaSuccess) return cuda_refusal(who, "count", sc.e);
        for (uint32_t t = 0; t < n_src; t++) df_src[t] += df_part[p][t];
        // ---- rules 2-4: per new document its length and its stored payload ----
#pragma omp parallel for schedule(static) num_threads(bm25x_host_threads(0))
        for (uint32_t d = 0; d < pt.n; d++) {
            const uint32_t nd = smap[pt.first + d];
            if (nd != BM25X_DOC_INF) {
                len[nd] = cnt[d];
                memcpy(&pay[(size_t)nd * 3], &spay[(size_t)d * 3], 6);
            }
        }
    }
    for (uint32_t o = 0; o < NG; o++)
        if (gmap[o] != BM25X_DOC_INF) {
            len[gmap[o]] = s.len[o];
            memcpy(&pay[(size_t)gmap[o] * 3], &s.payload[(size_t)o * 3], 6);
        }
    // ---- rule 6: the vocabulary ----
    std::vector<uint32_t> src_of;  // new term -> source term
    if (keyed) {
        for (uint32_t t = 0; t < n_src; t++)
            if (df_src[t]) src_of.push_back(t);
        std::sort(src_of.begin(), src_of.end(), key_less);
    } else {
        src_of.resize(n_src);
        for (uint32_t t = 0; t < n_src; t++) src_of[t] = t;
    }
    const uint32_t TN = (uint32_t)src_of.size();
    std::vector<uint32_t> df(TN), tmap(n_src, BM25X_TERM_MISSING);
    std::vector<uint8_t> keys(keyed ? (size_t)TN * 16 : 0);
    uint64_t P = 0, sum_len = 0;
    for (uint32_t j = 0; j < TN; j++) {
        df[j] = df_src[src_of[j]];
        tmap[src_of[j]] = j;
        P += df[j];
        if (keyed) memcpy(&keys[(size_t)j * 16], key_of(src_of[j]), 16);
    }
    for (uint32_t d = 0; d < N; d++) sum_len += len[d];
    // ---- rules 5 and 7: ONE set of statistics for the new segment; per part that keeps a document, a new handle on its
    // device scoring with them, its survivors spliced into it, then what every index derives from them ----
    const double k1 = sealed.home().k1, b = sealed.home().b;
    const Stats st(N, sum_len, df.data(), TN, k1, b);
    std::unique_ptr<bm25x_sharded_index, void (*)(bm25x_sharded_index *)> sx(new bm25x_sharded_index(),
                                                                             bm25x_sharded_destroy);
    sx->bounds.push_back(0);
    for (uint32_t p = 0; p < NP; p++) {
        const uint32_t lo = new_lo[p], n = new_lo[p + 1] - lo;
        if (!n) continue;  // a part left without a document is dropped
        std::vector<uint32_t> dfp(TN);
        uint64_t Pp = 0;
        for (uint32_t j = 0; j < TN; j++) Pp += dfp[j] = df_part[p][src_of[j]];
        // (the term keys once, with the new shard 0)
        BuildMeta m{n, TN, len.data() + lo, pay.data() + (size_t)lo * 3, keyed && sx->shards.empty() ? keys.data() : nullptr,
                    k1, b, dfp.data(), Pp};
        IndexGuard ix;
        Scratch &sc = *scs[p];
        int rc = index_begin(m, &st, parts[p].h->device, ix);
        if (rc == BM25X_OK) rc = splice_finish(sc, who, ix.get(), sc.up(src_of.data(), TN), srcs[p]);
        if (rc != BM25X_OK) return rc;
        sx->shards.push_back(ix.release());
        sx->bounds.push_back(lo + n);
    }
    sx->n_shards = (uint32_t)sx->shards.size();
    sx->n_docs = N;
    sx->n_terms = TN;
    sx->n_post = P;
    sx->k1 = k1;
    sx->b = b;
    sx->h_df = std::move(df);
    sx->sum_len = sum_len;
    sx->avgdl = st.avgdl;
    a->n_growing = NG;
    a->n_source_terms = n_src;
    if (a->sealed_map) std::copy(smap.begin(), smap.end(), a->sealed_map);
    if (a->growing_map) std::copy(gmap.begin(), gmap.end(), a->growing_map);
    if (a->term_map) std::copy(tmap.begin(), tmap.end(), a->term_map);
    {
        // the record a rebind to this result needs; a seal that a rebind overtook leaves none (its ordinals are gone)
        std::lock_guard<std::mutex> lock(g->mu);
        if (g->bind == bind) {
            g->last_seal.serial = g->sharded ? sx->serial : sx->shards[0]->serial;
            g->last_seal.n_growing = NG;
            g->last_seal.gmap = std::move(gmap);
            g->last_seal.tmap = std::move(tmap);
        }
    }
    *out = sx.release();
    return BM25X_OK;
}

extern "C" int bm25x_growing_seal(bm25x_growing_segment *g, bm25x_seal_args *a, bm25x_index **out) {
    const char *who = "bm25x_growing_seal";
    if (!g || !a || !out || (a->n_new_keys && !a->new_keys)) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    if (g->sharded) {
        bm25x_set_error("%s: the segment was opened over a document-sharded index: seal it with bm25x_growing_seal_sharded",
                        who);
        return BM25X_ERR_INVALID;
    }
    bm25x_sharded_index *sx = nullptr;
    const int rc = seal_segment(who, g, a, &sx);
    if (rc != BM25X_OK) return rc;
    *out = sx->shards[0];  // one part: one shard, detached from its container
    sx->shards.clear();
    bm25x_sharded_destroy(sx);
    return BM25X_OK;
}

extern "C" int bm25x_growing_seal_sharded(bm25x_growing_segment *g, bm25x_seal_args *a, bm25x_sharded_index **out) {
    const char *who = "bm25x_growing_seal_sharded";
    if (!g || !a || !out || (a->n_new_keys && !a->new_keys)) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    *out = nullptr;
    if (!g->sharded) {
        bm25x_set_error("%s: the segment was opened over an unsharded index: seal it with bm25x_growing_seal", who);
        return BM25X_ERR_INVALID;
    }
    return seal_segment(who, g, a, out);
}

// ---- the rebind (DESIGN §4.5): the segment goes on over the index its latest seal built.  The ordinals the seal folded
// in leave it, the carried ones are renumbered from 0 and their elements translated to the new vocabulary; the carried
// postings of the new handle come from the current handle on the device and from the host's dormant list ----

// How a carried element's term is translated: the segment's numbering of its terms.
enum class Numbering { KEYLESS, OWNED, CALLER };

static int rebind_segment(const char *who, bm25x_growing_segment *g, const SealedSide &side, uint64_t serial,
                          bm25x_rebind_args *a) {
    std::unique_lock<std::mutex> numbering(g->num_mu);  // ordered with the tsvector inserts, which read the binding
    std::unique_lock<std::mutex> lock(g->mu);
    const SealRecord &rec = g->last_seal;
    if (!rec.serial) {
        bm25x_set_error("%s: no seal to rebind to (no seal of the segment has succeeded since it was opened or last "
                        "rebound)", who);
        return BM25X_ERR_INVALID;
    }
    if (rec.serial != serial) {
        bm25x_set_error("%s: the index is not the one the segment's latest seal returned", who);
        return BM25X_ERR_INVALID;
    }
    int rc = growing_refresh_locked(g);
    if (rc != BM25X_OK) return rc;
    const Binding &ob = *g->bind;
    const uint32_t NG = rec.n_growing, N = g->n_docs(), NC = N - NG;
    const uint32_t To = ob.sealed.n_terms(), Tn = side.n_terms(), K = g->n_keys();
    const std::vector<uint32_t> &ndf = side.df();
    const Numbering kind = g->owns_keys ? Numbering::OWNED : ob.sealed.keys().empty() ? Numbering::KEYLESS
                                                                                       : Numbering::CALLER;
    const uint32_t n_old = std::max(To + K, g->term_end);  // the old source-term space
    // a term the new handle holds: one with postings in the new index (a growing handle leaves the others out)
    auto live_new = [&](uint32_t u) { return u < Tn && ndf[u] != 0; };
    const bm25x_index *cur = NC ? g->cur.get() : nullptr;
    const int od = ob.device, nd = side.home().device;
    const bool same = od == nd;
    // ---- the carried ordinals: old o >= NG becomes o - NG; a folded or deleted ordinal gives no posting ----
    std::vector<uint8_t> gone(N);
    std::vector<uint32_t> cmap(N);
    for (uint32_t o = 0; o < N; o++) {
        gone[o] = o < NG || g->deleted[o];
        cmap[o] = o < NG ? BM25X_DOC_INF : o - NG;
    }
    const std::vector<uint32_t> bits = deleted_bitmap(gone);
    // ---- the current handle's carried survivors per term (k_splice_count), on its device ----
    Scratch sco(od);
    sco.e = cudaSetDevice(od);
    SpliceSources hs{};
    std::vector<uint32_t> hcnt;
    if (cur) {
        hs.s[0] = handle_source(cur, sco.up(bits.data(), bits.size()), sco.up(cmap.data(), N));
        hcnt = splice_count(sco, cur->sm_count, To, hs);
        if (sco.e != cudaSuccess) return cuda_refusal(who, "count", sco.e);
    }
    hcnt.resize(To, 0);
    std::vector<uint32_t> dcnt(n_old, 0);  // the carried dormant postings per term
    for (size_t i = 0; i < g->dorm_doc.size(); i++)
        if (!gone[g->dorm_doc[i]]) dcnt[g->dorm_term[i]]++;
    // ---- the translation of every old term a carried posting holds ----
    std::vector<uint32_t> xl(n_old, BM25X_TERM_MISSING);
    std::vector<uint8_t> owned;  // OWNED: the carried keys the new vocabulary lacks, ascending
    if (kind == Numbering::KEYLESS) {
        for (uint32_t t = 0; t < n_old; t++) xl[t] = t;
    } else if (kind == Numbering::CALLER) {
        for (uint32_t t = 0; t < n_old && t < (uint32_t)rec.tmap.size(); t++) xl[t] = rec.tmap[t];
    } else {
        const uint8_t *okeys = ob.sealed.keys().data(), *nkeys = side.keys().data();
        auto key_of = [&](uint32_t t) { return t < To ? okeys + (size_t)t * 16 : g->new_keys.data() + (size_t)(t - To) * 16; };
        std::vector<uint32_t> lack;
        for (uint32_t t = 0; t < n_old; t++) {
            if (!(t < To ? hcnt[t] : 0) && !dcnt[t]) continue;
            xl[t] = key_ordinal(nkeys, Tn, key_of(t));
            if (xl[t] == BM25X_TERM_MISSING) lack.push_back(t);
        }
        std::sort(lack.begin(), lack.end(), [&](uint32_t x, uint32_t y) { return memcmp(key_of(x), key_of(y), 16) < 0; });
        if ((uint64_t)Tn + lack.size() >= BM25X_TERM_MISSING) {
            bm25x_set_error("%s: more than %u term ordinals (%u is BM25X_TERM_MISSING)", who, BM25X_TERM_MISSING,
                            BM25X_TERM_MISSING);
            return BM25X_ERR_UNSUPPORTED;
        }
        for (uint32_t r = 0; r < (uint32_t)lack.size(); r++) {
            xl[lack[r]] = Tn + r;
            owned.insert(owned.end(), key_of(lack[r]), key_of(lack[r]) + 16);
        }
    }
    // ---- down: the carried postings of the handle's terms the new handle does not keep (across devices: all of them),
    // compacted on the device by k_splice_emit at the offsets of their scan, then one download ----
    std::vector<uint64_t> down_off((size_t)To + 1, 0);
    for (uint32_t t = 0; t < To; t++)
        down_off[(size_t)t + 1] = down_off[t] + (!same || !live_new(xl[t]) ? hcnt[t] : 0);
    const uint64_t D = down_off[To];
    std::vector<uint32_t> dn_term(D), dn_doc(D), dn_tf(D);
    if (D) {
        const uint64_t *d_off = sco.up(down_off.data(), down_off.size());
        uint32_t *d_doc = sco.alloc<uint32_t>(D), *d_tf = sco.alloc<uint32_t>(D);
        if (sco.e == cudaSuccess) {
            k_splice_emit<<<splice_grid(To, cur->sm_count), 256>>>(To, hs.s[0], d_off, d_doc, d_tf);
            sco.e = cudaGetLastError();
        }
        if (sco.e == cudaSuccess) sco.e = cudaMemcpy(dn_doc.data(), d_doc, sizeof(uint32_t) * D, cudaMemcpyDeviceToHost);
        if (sco.e == cudaSuccess) sco.e = cudaMemcpy(dn_tf.data(), d_tf, sizeof(uint32_t) * D, cudaMemcpyDeviceToHost);
        if (sco.e != cudaSuccess) return cuda_refusal(who, "carry", sco.e);
        for (uint32_t t = 0; t < To; t++)
            std::fill(dn_term.begin() + down_off[t], dn_term.begin() + down_off[(size_t)t + 1], t);
    }
    // ---- the carried postings on the host (down, then dormant; a term has postings in one of them only): a keyed
    // caller-numbered term without a new ordinal is refused, a term the new handle keeps goes up, any other stays
    // dormant under its new ordinal ----
    if (kind == Numbering::CALLER) {
        uint64_t worst = ~0ull;  // (carried ordinal, old term) of the first carried posting without a new ordinal
        for (uint64_t i = 0; i < D; i++)
            if (xl[dn_term[i]] == BM25X_TERM_MISSING) worst = std::min(worst, (uint64_t)dn_doc[i] << 32 | dn_term[i]);
        for (size_t i = 0; i < g->dorm_doc.size(); i++) {
            const uint32_t o = g->dorm_doc[i], t = g->dorm_term[i];
            if (!gone[o] && xl[t] == BM25X_TERM_MISSING) worst = std::min(worst, (uint64_t)(o - NG) << 32 | t);
        }
        if (worst != ~0ull) {
            const uint32_t o = (uint32_t)(worst >> 32) + NG, t = (uint32_t)worst;
            if (t >= rec.tmap.size())
                bm25x_set_error("%s: growing ordinal %u holds term ordinal %u >= n_source_terms=%u of the seal: no key is "
                                "known for it (insert the document again)", who, o, t, (uint32_t)rec.tmap.size());
            else
                bm25x_set_error("%s: growing ordinal %u holds term ordinal %u, whose key vanished in the seal (insert the "
                                "document again)", who, o, t);
            return BM25X_ERR_INVALID;
        }
    }
    std::vector<uint32_t> up_term, up_doc, up_tf, nd_term, nd_doc, nd_tf;
    bool big = false;
    auto route = [&](uint32_t t, uint32_t d, uint32_t f) {
        const uint32_t u = xl[t];
        if (live_new(u)) {
            big |= f >= (1u << 24);
            up_term.push_back(t);
            up_doc.push_back(d);
            up_tf.push_back(f);
        } else {
            nd_term.push_back(u);
            nd_doc.push_back(d);
            nd_tf.push_back(f);
        }
    };
    for (uint64_t i = 0; i < D; i++) route(dn_term[i], dn_doc[i], dn_tf[i]);
    for (size_t i = 0; i < g->dorm_doc.size(); i++)
        if (!gone[g->dorm_doc[i]]) route(g->dorm_term[i], g->dorm_doc[i] - NG, g->dorm_tf[i]);
    if (big) {  // what the insert of the restated documents refuses
        bm25x_set_error("%s: term frequency >= 2^24 is not supported by the packed posting layout", who);
        return BM25X_ERR_UNSUPPORTED;
    }
    // ---- the new handle: new term u from old term src_of[u], its survivors in the handle (same device) and those that
    // came up, opened with the new statistics on the new home device ----
    const auto nb = std::make_shared<Binding>(side);
    IndexGuard ix;
    if (NC) {
        std::unique_ptr<Scratch> other;
        Scratch &scn = same ? sco : *(other = std::make_unique<Scratch>(nd));
        scn.e = cudaSetDevice(nd);
        std::vector<uint32_t> src_of(Tn, BM25X_TERM_MISSING), df(Tn, 0), ucnt(n_old, 0);
        for (uint32_t t : up_term) ucnt[t]++;
        uint64_t P = 0;
        for (uint32_t t = 0; t < n_old; t++)
            if (live_new(xl[t])) {
                src_of[xl[t]] = t;
                P += df[xl[t]] = (same && t < To ? hcnt[t] : 0) + ucnt[t];
            }
        const std::vector<uint32_t> zero(((size_t)NC + 31) / 32, 0);
        SpliceSources src{};
        if (same) src.s[0] = hs.s[0];
        src.s[1] = grouped_source(scn, n_old, up_term, up_doc, up_tf, scn.up(zero.data(), zero.size()), nullptr);
        if (scn.e != cudaSuccess) return cuda_refusal(who, "carry", scn.e);
        const std::vector<uint8_t> &keys = side.keys();
        BuildMeta m{NC, Tn, g->norm_form ? g->doc_len.data() + NG : nullptr, g->payload.data() + (size_t)NG * 3,
                    keys.empty() ? nullptr : keys.data(), side.home().k1, side.home().b, df.data(), P};
        m.fieldnorm = g->norm_form ? nullptr : g->fieldnorm.data() + NG;
        rc = index_begin(m, &nb->stats, nd, ix);
        if (rc == BM25X_OK) rc = splice_finish(scn, who, ix.get(), scn.up(src_of.data(), Tn), src);
        if (rc != BM25X_OK) return rc;
        growing_options(ix.get(), side);
    }
    // ---- commit: nothing is refused from here on ----
    const uint32_t NN = side.n_docs();
    uint32_t n_late = 0;
    if (a->late_deleted) memset(a->late_deleted, 0, ((size_t)NN + 7) / 8);
    for (uint32_t o = 0; o < NG; o++)
        if (g->deleted[o] && rec.gmap[o] != BM25X_DOC_INF) {
            n_late++;
            if (a->late_deleted) a->late_deleted[rec.gmap[o] >> 3] |= (uint8_t)(1u << (rec.gmap[o] & 7u));
        }
    a->n_late_deleted = n_late;
    a->n_folded = NG;
    a->n_carried = NC;
    g->fieldnorm.erase(g->fieldnorm.begin(), g->fieldnorm.begin() + NG);
    if (g->norm_form == 1) g->doc_len.erase(g->doc_len.begin(), g->doc_len.begin() + NG);
    if (g->norm_form == 0) g->sum_tf.erase(g->sum_tf.begin(), g->sum_tf.begin() + NG);
    g->payload.erase(g->payload.begin(), g->payload.begin() + (size_t)NG * 3);
    g->deleted.erase(g->deleted.begin(), g->deleted.begin() + NG);
    g->n_deleted = (uint32_t)std::count(g->deleted.begin(), g->deleted.end(), (uint8_t)1);
    // the dormant postings as one insert of the carried documents appends them: by document, then by term
    std::vector<uint32_t> perm(nd_term.size());
    for (uint32_t i = 0; i < (uint32_t)perm.size(); i++) perm[i] = i;
    std::sort(perm.begin(), perm.end(), [&](uint32_t x, uint32_t y) {
        return nd_doc[x] != nd_doc[y] ? nd_doc[x] < nd_doc[y] : nd_term[x] < nd_term[y];
    });
    g->dorm_term.resize(perm.size());
    g->dorm_doc.resize(perm.size());
    g->dorm_tf.resize(perm.size());
    for (size_t i = 0; i < perm.size(); i++) {
        g->dorm_term[i] = nd_term[perm[i]];
        g->dorm_doc[i] = nd_doc[perm[i]];
        g->dorm_tf[i] = nd_tf[perm[i]];
    }
    // the carried ordinals >= n_terms(new), in the order they first come in the carried documents (every one of them is
    // dormant; a keyed caller-numbered segment has none)
    g->new_terms.clear();
    g->new_seen.clear();
    g->term_end = 0;
    for (uint32_t u : g->dorm_term)
        if (u >= Tn && g->new_seen.insert(u).second) {
            g->new_terms.push_back(u);
            g->term_end = std::max(g->term_end, u + 1);
        }
    if (kind == Numbering::OWNED) {
        g->new_keys = std::move(owned);
        g->key_ord.clear();
        for (uint32_t r = 0; r < g->n_keys(); r++) g->key_ord.emplace(key16(&g->new_keys[(size_t)r * 16]), Tn + r);
    }
    if (ix) g->cur.reset(ix.release(), IndexDestroy());
    else g->cur.reset();
    g->last_seal = SealRecord();
    std::shared_ptr<Binding> old = std::move(g->bind);
    g->bind = nb;
    // ---- the old binding's holders finish with it; its last one fires `released` ----
    std::promise<void> released;
    std::future<void> done = released.get_future();
    old->released = &released;
    lock.unlock();
    numbering.unlock();
    old.reset();
    done.wait();
    return BM25X_OK;
}

extern "C" int bm25x_growing_rebind(bm25x_growing_segment *g, bm25x_index *sealed, bm25x_rebind_args *a) {
    const char *who = "bm25x_growing_rebind";
    if (!g || !sealed || !a) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    if (g->sharded) {
        bm25x_set_error("%s: the segment was opened over a document-sharded index: rebind it with "
                        "bm25x_growing_rebind_sharded", who);
        return BM25X_ERR_INVALID;
    }
    SealedSide side;
    side.ix = sealed;
    return rebind_segment(who, g, side, sealed->serial, a);
}

extern "C" int bm25x_growing_rebind_sharded(bm25x_growing_segment *g, bm25x_sharded_index *sealed, bm25x_rebind_args *a) {
    const char *who = "bm25x_growing_rebind_sharded";
    if (!g || !sealed || !a) {
        bm25x_set_error("%s: null argument", who);
        return BM25X_ERR_INVALID;
    }
    if (!g->sharded) {
        bm25x_set_error("%s: the segment was opened over an unsharded index: rebind it with bm25x_growing_rebind", who);
        return BM25X_ERR_INVALID;
    }
    SealedSide side;
    side.sx = sealed;
    return rebind_segment(who, g, side, sealed->serial, a);
}
