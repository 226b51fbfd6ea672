"""Exact BM25 reference whose cost is in postings, not documents: for corpora whose doc ids span the 32-bit range.

util_index.restate and the oracle allocate per-document arrays (the oracle's accumulator, the synthetic payload of every
document), which do not fit at n_docs = 2^32 - 2.  Here a query touches only its terms' postings: each document's score
is summed in ascending term order from 0.0 with the product's operation order (tf * s0) / (tf + s1[fn]), so the f64 sum
runs left to right as the oracle's does, then the prefilter bitmap, then (score desc, doc asc).  s0 / s1 come from the
oracle's Cache (util_index.cache); the posting-side arrays of a handle come from util_index.restate_postings.  Pinned
against OracleIndex.search_exhaustive and util_index.restate by tests/test_sparse_reference.py.

high_id_corpus() builds the corpus of tests/test_gpu_zy_high_doc_ids.py: a few hundred thousand postings on documents
placed on purpose across the 32-bit id space; high_id_queries() the queries over it, and need() skips a test whose index
does not fit in the host or device memory available."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest

from util_cuda import cudart
from util_index import cache, ctid, restate_postings
from util_parity import query_csr

DOC_INF = 0xFFFFFFFF
MAX_N_DOCS = 0xFFFFFFFE  # the largest n_docs the library accepts; the largest doc id is MAX_N_DOCS - 1


def norms_present(fieldnorm, chunk=1 << 26):
    """Distinct values of a (possibly 4 GB) u8 array, chunk by chunk."""
    seen = np.zeros(256, dtype=bool)
    for i in range(0, len(fieldnorm), chunk):
        seen |= np.bincount(fieldnorm[i:i + chunk], minlength=256) > 0
    return np.flatnonzero(seen)


class SparseReference:
    """One index's exact rankings and posting-side arrays.  fieldnorm: per-document u8 array indexed by doc id (length
    n_docs); or post_fn: the fieldnorm of each posting's document, with norms = the distinct fieldnorms of all documents.
    stat = (n_docs, df[n_terms], avgdl) to score with instead of the corpus' own (a growing segment uses its sealed
    segment's)."""

    def __init__(self, orc, n_docs, post_off, post_doc, post_tf, k1, b, sum_len, fieldnorm=None, post_fn=None, norms=None,
                 stat=None):
        self.orc, self.n_docs, self.k1, self.b, self.sum_len, self.stat = orc, int(n_docs), float(k1), float(b), int(sum_len), stat
        self.off = np.asarray(post_off, dtype=np.int64)
        self.doc = np.asarray(post_doc, dtype=np.uint32)
        self.tf = np.asarray(post_tf, dtype=np.uint32)
        assert len(self.doc) == self.off[-1] and (len(self.doc) == 0 or int(self.doc.max()) < self.n_docs)
        self.df = np.diff(self.off)
        if fieldnorm is not None:
            assert len(fieldnorm) == self.n_docs
            self.post_fn = np.asarray(fieldnorm[self.doc.astype(np.int64)], dtype=np.uint8)
            self.norms = norms if norms is not None else norms_present(fieldnorm)
        else:
            self.post_fn, self.norms = np.asarray(post_fn, dtype=np.uint8), norms
        avgdl = float(stat[2]) if stat is not None else float(self.sum_len) / float(self.n_docs)
        s0, s1 = cache(orc, stat[0] if stat is not None else self.n_docs, stat[1] if stat is not None else self.df, k1, b,
                       avgdl)
        term = np.repeat(np.arange(len(self.df)), self.df)
        tfd = self.tf.astype(np.float64)
        self.score = (tfd * s0[term]) / (tfd + s1[self.post_fn])

    def arrays(self):
        """post, post_off, df, blk_off, blk, s0d/s0f/s1d/s1f, ubd, blk_ub, pdoc, champ, champ_off, s1f_min and the layout's
        scalars, as util_index.restate gives them."""
        return restate_postings(self.orc, self.n_docs, self.off, self.doc, self.tf, self.post_fn, self.norms, self.k1,
                                self.b, self.sum_len, stat=self.stat)

    def live_terms(self, terms):
        """The canonical query (search.rs:55-62): distinct known terms with df > 0, ascending."""
        t = np.unique(np.asarray(terms, dtype=np.int64))
        t = t[(t >= 0) & (t < len(self.df))]
        return t[self.df[t] > 0]

    def search(self, terms, k, allow=None):
        """Top-k rows: doc (u32), score64, score (f32 of score64), payload ([n, 3] synthetic ctid of the ids), n."""
        q = self.live_terms(terms)
        lists = [(self.doc[self.off[t]:self.off[t + 1]], self.score[self.off[t]:self.off[t + 1]]) for t in q]
        docs = np.unique(np.concatenate([d for d, _ in lists])) if lists else np.zeros(0, np.uint32)
        acc = np.zeros(len(docs))
        for d, s in lists:  # ascending term order: acc = ((0.0 + s_t0) + s_t1) + ...
            np.add.at(acc, np.searchsorted(docs, d), s)
        if allow is not None and len(docs):
            d64 = docs.astype(np.int64)
            keep = (np.asarray(allow)[d64 >> 3] >> (d64 & 7)) & 1
            docs, acc = docs[keep == 1], acc[keep == 1]
        order = np.lexsort((docs, -acc))[:k]
        return SimpleNamespace(doc=docs[order].astype(np.uint32), score64=acc[order], score=acc[order].astype(np.float32),
                               payload=ctid(docs[order]), n=len(order))


def assert_rows(res, ref, terms_of, k, what, allow=None, payload_of=ctid):
    """Every row of a search result (dict of search_batch) equal to the reference: ids, f64 and f32 scores, payload (when
    the result holds one), and the empty slots (0xFFFFFFFF, zero scores)."""
    for i, terms in enumerate(terms_of):
        want = ref.search(terms, k, allow=allow)
        n = int(res["n"][i])
        assert n == want.n, f"{what} q{i}: n {n} != {want.n}"
        if not np.array_equal(res["doc"][i, :n], want.doc):
            bad = np.flatnonzero(res["doc"][i, :n] != want.doc)[:4]
            raise AssertionError(f"{what} q{i} k={k}: ids differ at ranks {bad.tolist()}: got {res['doc'][i, bad].tolist()} "
                                 f"want {want.doc[bad].tolist()}")
        assert np.array_equal(res["score64"][i, :n], want.score64), f"{what} q{i}: f64 scores"
        assert np.array_equal(res["score"][i, :n], want.score), f"{what} q{i}: f32 scores"
        assert np.all(res["doc"][i, n:] == DOC_INF) and np.all(res["score64"][i, n:] == 0.0), f"{what} q{i}: empty slots"
        if res.get("payload") is not None:
            assert np.array_equal(res["payload"][i, :n], payload_of(want.doc)), f"{what} q{i}: payload"


# ---- the high-id corpus ----

T31 = 1 << 31
FN_EMPTY = 20          # fieldnorm of every document without postings (nearly all of them)
FN_TIE = 24            # fieldnorm of every member of a tie group
N_HEAD, N_DENSE, N_FILL = 4, 6, 120


def high_id_corpus(n_docs, seed=0x1D5):
    """Term-major CSR over ids spread across [0, n_docs), n_docs close to 2^32:
    - documents at [0, 2^16), the 3000 ids around 2^31 (2^31 - 1, 2^31, 2^31 + 1 included), near 3 * 2^30, all of the
      top 2048 ids (n_docs - 1 included) and ~90k scattered over the whole range;
    - head terms (df ~ 40k: pruning, probes, blocks across 2^31; three of them match > 65 535 documents together);
    - tie terms: tf 1 on documents of one fieldnorm on both sides of 2^31 and at both ends of the range, behind a few
      tf 2 postings, so that the champion cut (128) and the limits 128 / 129 / 224 fall inside a tie group past 2^31;
    - dense terms: hundreds of postings each inside the top 2048 ids (dense windows that start there);
    - a pad term whose last posting is n_docs - 1 with df = 1 (mod 4);
    - a wide term: one full block with a gap >= 2^31 (bit width 32) and a tail of ids >= 2^31 with a gap >= 2^24 (byte
      width 4);
    - filler terms of every df from 1 to a few thousand.
    Returns a namespace: n_docs, post_off, post_doc, post_tf, live (ids with postings), live_fn (their fieldnorms), the
    term ids of each kind, and sum_len (every document's length, the empty ones at FN_EMPTY's length)."""
    N = int(n_docs)
    rng = np.random.default_rng(seed)
    top = np.arange(N - 2048, N, dtype=np.int64)
    mid = np.arange(T31 - 1500, T31 + 1500, dtype=np.int64)
    low = np.arange(3000, dtype=np.int64) * 21
    q3 = 3 * (1 << 30) - (1 << 20) + np.sort(rng.choice(1 << 21, 2000, replace=False))
    scatter = np.sort(rng.choice(N, 90000, replace=False)).astype(np.int64)
    live = np.unique(np.concatenate([low, mid, q3, top, scatter]))
    live_fn = rng.choice(np.array([12, 18, FN_TIE, 30, 41, 57], np.uint8), len(live))
    idx = lambda ids: np.searchsorted(live, ids)
    lists, kinds = [], {}

    def add(kind, docs, tfs):
        docs = np.asarray(docs, np.int64)
        assert np.all(np.diff(docs) > 0) and np.all(np.isin(docs, live))
        kinds.setdefault(kind, []).append(len(lists))
        lists.append((docs, np.asarray(tfs, np.int64)))

    for _ in range(N_HEAD):
        d = np.sort(rng.choice(live, int(0.4 * len(live)), replace=False))
        add("head", d, rng.integers(1, 7, len(d)))
    # tie groups: members share FN_TIE and tf 1; a few tf 2 postings rank first
    below = np.concatenate([low[:40], mid[mid < T31][-60:]])              # 100 ids below 2^31 (2^31 - 1 included)
    above = np.concatenate([mid[mid >= T31][:150], q3[:50], top[:100]])   # 300 ids >= 2^31 (2^31, 2^31 + 1 included)
    for s in range(2):
        d = np.unique(np.concatenate([below, above, rng.choice(scatter, 30 * s, replace=False)]))
        tf = np.ones(len(d), np.int64)
        tf[rng.choice(len(d), 20 - 10 * s, replace=False)] = 2
        live_fn[idx(d)] = FN_TIE
        add("tie", d, tf)
    d = np.concatenate([low[:64], [T31 - 1, T31, T31 + 1], top[-64:]])       # both ends and the middle, one tie
    live_fn[idx(d)] = FN_TIE
    add("tie", d, np.ones(len(d)))
    for _ in range(N_DENSE):
        d = np.sort(rng.choice(top, int(rng.integers(300, 900)), replace=False))
        add("dense", d, rng.integers(1, 5, len(d)))
    add("pad", top[-301:], rng.integers(1, 4, 301))                           # ends at N - 1, df = 1 (mod 4)
    wide = np.concatenate([[low[7]], mid[mid >= T31][200:327], q3[100:120], top[200:220]])
    add("wide", wide, rng.integers(1, 9, len(wide)))
    for i in range(N_FILL):
        n = int(min(len(live), 1 + rng.integers(0, 40) ** 2 * 3)) if i else 1
        d = np.sort(rng.choice(live, n, replace=False))
        add("fill", d, rng.integers(1, 12, n))

    off = np.zeros(len(lists) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d, _ in lists])
    post_doc = np.concatenate([d for d, _ in lists]).astype(np.uint32)
    post_tf = np.concatenate([t for _, t in lists]).astype(np.uint32)
    return SimpleNamespace(n_docs=N, post_off=off, post_doc=post_doc, post_tf=post_tf, live=live, live_fn=live_fn,
                           kinds=kinds, n_terms=len(lists))


def sum_len_of(orc, c):
    """Σ of every document's length: FN_EMPTY's length for the documents without postings."""
    L = orc.lib()
    length = np.array([L.orc_fieldnorm_to_length(f) for f in range(256)], dtype=np.int64)
    return int(length[c.live_fn].sum()) + (c.n_docs - len(c.live)) * int(length[FN_EMPTY])


def full_fieldnorm(c):
    """The per-document fieldnorm array (n_docs bytes)."""
    fn = np.full(c.n_docs, FN_EMPTY, dtype=np.uint8)
    fn[c.live] = c.live_fn
    return fn


def reference(orc, c, k1, b):
    """SparseReference of the corpus, from its documents with postings only."""
    norms = np.unique(np.append(c.live_fn, FN_EMPTY)) if len(c.live) < c.n_docs else np.unique(c.live_fn)
    post_fn = c.live_fn[np.searchsorted(c.live, c.post_doc.astype(np.int64))]
    return SparseReference(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, k1, b, sum_len_of(orc, c), post_fn=post_fn,
                           norms=norms)


# ---- the high-id indexes ----

N_A = MAX_N_DOCS - 64       # index A: room for a growing segment of 64 documents, ids up to 0xFFFFFFFD
K1, B = 1.2, 0.75


def need(host_gb, dev_gb, what):
    import psutil
    free, total = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert cudart().cudaMemGetInfo(ctypes.byref(free), ctypes.byref(total)) == 0
    host = psutil.virtual_memory().available
    if host < host_gb * 1e9 or free.value < dev_gb * 1e9:
        pytest.skip(f"{what} needs {host_gb} GB of host and {dev_gb} GB of free device memory "
                    f"({host / 1e9:.0f} GB / {free.value / 1e9:.0f} GB available)")


def peak_host_gb():
    import resource
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6


def high_id_queries(c, seed):
    """Queries of 1, 2, 3, 4, 5-8, 9-16, 17-32 and 33-64 live terms over the corpus' kinds of terms."""
    k = c.kinds
    rng = np.random.default_rng(seed)
    rand = lambda n: rng.choice(c.n_terms, n, replace=False)
    qs = [[t] for t in k["tie"] + k["dense"][:2] + k["pad"] + k["wide"] + k["head"][:1] + k["fill"][-2:]]
    qs += [[k["tie"][0], k["dense"][0]], [k["head"][0], k["tie"][1]], k["dense"][:2], [k["pad"][0], k["tie"][2]]]
    qs += [k["dense"][:3], [k["head"][0], k["head"][1], k["tie"][0]], k["tie"]]
    qs += [k["dense"][:4], k["pad"] + k["dense"][:2] + k["wide"], k["tie"] + k["pad"]]
    qs += [k["dense"] + k["pad"], k["head"] + k["tie"], list(rand(5)), list(rand(8))]
    qs += [k["dense"] + k["tie"] + list(rand(3)), list(rand(16)), list(rand(17)), list(rand(32)), list(rand(33)),
           list(rand(64))]
    qs = [np.unique(np.asarray(q, np.uint32)) for q in qs]
    q_off, q_terms = query_csr(qs)
    return q_off, q_terms, qs


class Prefix:
    """SparseReference.search at one limit per (query, bitmap): every smaller limit's rows are a prefix."""

    def __init__(self, ref, kmax):
        self.ref, self.kmax, self.memo = ref, kmax, {}

    def search(self, terms, k, allow=None):
        key = (np.asarray(terms, np.uint32).tobytes(), id(allow))
        if key not in self.memo:
            self.memo[key] = self.ref.search(terms, self.kmax, allow=allow)
        r = self.memo[key]
        n = min(k, r.n)
        return SimpleNamespace(doc=r.doc[:n], score64=r.score64[:n], score=r.score[:n], payload=r.payload[:n], n=n)
