"""The two references of bm25x_evaluate_tsvectors (`<&>` from tsvectors in one call), shared by its GPU test files:

(a) the oracle: OracleIndex.evaluate over the restated casts (util_tsvector.cast over bm25x_intern), each key taken to its
    ordinal in the index's sorted vocabulary, the document's unknown keys numbered past it in key order (they count in
    Document::length and never score), each row sorted by ordinal;
(b) the four-step route a caller takes without it: the document cast on the GPU, every key looked up on the host, the
    unknown keys numbered past n_terms in key order and every row re-sorted by ordinal, the queries through
    tsvector_queries (TERM_MISSING dropped), each query repeated for its pairs, and bm25x_evaluate_batch."""
import ctypes as C

import numpy as np

from util_documents import key_words
from util_evaluate import oracle_csr
from util_tsvector import cast

SEED = bytes(range(32))


def _bm(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


def ordinals(vocab, keys):
    """Each key's ordinal in the sorted vocabulary ([T, 16]), or -1 when absent."""
    vh, vl = key_words(vocab)
    kh, kl = key_words(keys)
    T = len(vh)
    # the vocabulary as one sortable array of (hi, lo) pairs
    v = np.empty(T, [("h", ">u8"), ("l", ">u8")])
    v["h"], v["l"] = vh, vl
    k = np.empty(len(kh), v.dtype)
    k["h"], k["l"] = kh, kl
    at = np.searchsorted(v, k)
    hit = at < T
    hit[hit] = v[at[hit]] == k[hit]
    return np.where(hit, at, -1).astype(np.int64)


def sorted_rows(off, ordinal, tf, n_terms, unknown_rank):
    """The rows off[i]:off[i+1] with unknown keys (ordinal < 0) as n_terms + their rank, each row sorted by ordinal:
    (terms u32, tfs u32 or None) in the same offsets."""
    o = ordinal.copy()
    o[o < 0] = n_terms + unknown_rank[o < 0]
    row = np.repeat(np.arange(len(off) - 1), np.diff(np.asarray(off, np.int64)))
    s = np.lexsort((o, row))
    return o[s].astype(np.uint32), None if tf is None else np.asarray(tf)[s].astype(np.uint32)


def pair_queries(q_off, q_terms, keep, pair_query, n):
    """The query rows with only the entries `keep` marks, sorted, repeated for the pairs: (off u32 [n+1], terms u32)."""
    q_off = np.asarray(q_off, np.int64)
    row = np.repeat(np.arange(len(q_off) - 1), np.diff(q_off))
    row, t = row[keep], np.asarray(q_terms)[keep].astype(np.int64)
    s = np.lexsort((t, row))
    row, t = row[s], t[s]
    k_off = np.zeros(len(q_off), np.int64)
    k_off[1:] = np.cumsum(np.bincount(row, minlength=len(q_off) - 1))
    pq = np.arange(n) if pair_query is None else np.asarray(pair_query, np.int64)
    lens = k_off[pq + 1] - k_off[pq]
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(lens)
    sel = np.repeat(k_off[pq] - off[:-1], lens) + np.arange(int(off[-1]))
    return off.astype(np.uint32), t[sel].astype(np.uint32)


def unknown_ranks(keys, ordinal):
    """The rank of each unknown key among the distinct unknown keys, in key order (0 for known keys)."""
    rank = np.zeros(len(keys), np.int64)
    miss = ordinal < 0
    if miss.any():
        h, l = key_words(keys[miss])
        u = np.empty(int(miss.sum()), [("h", ">u8"), ("l", ">u8")])
        u["h"], u["l"] = h, l
        _, inv = np.unique(u, return_inverse=True)
        rank[miss] = inv.reshape(-1)
    return rank


def oracle_pairs(m, vocab, n_terms, docs, queries, pair_query):
    """Reference (a)'s pairs as ordinal CSR arrays: (d_off, d_terms, d_tfs, q_off, q_terms), unknown query keys dropped."""
    bm = _bm(m)
    d_off, d_keys, d_tf = cast(bm.intern, SEED, docs)
    q_off, q_keys, _ = cast(bm.intern, SEED, queries, as_query=True)
    d_ord = ordinals(vocab, d_keys)
    dt, dtf = sorted_rows(d_off, d_ord, d_tf, n_terms, unknown_ranks(d_keys, d_ord))
    q_ord = ordinals(vocab, q_keys)
    p_off, p_terms = pair_queries(q_off, q_ord, q_ord >= 0, pair_query, len(d_off) - 1)
    return d_off.astype(np.uint32), dt, dtf, p_off, p_terms


def oracle_evaluate(m, oix, vocab, n_terms, docs, queries, pair_query=None):
    """Reference (a): the oracle's bm25::evaluate of every pair."""
    return oracle_csr(oix, *oracle_pairs(m, vocab, n_terms, docs, queries, pair_query))


def four_step_pairs(m, h, docs, queries, pair_query):
    """Reference (b)'s pairs as ordinal CSR arrays, through the GPU cast and the handle h (an Index or ShardedIndex)."""
    d_off, d_keys, d_tf = m.cast_tsvectors(SEED, **docs)
    n_terms = int(h.info().n_terms)
    ordinal = h.lookup_terms(d_keys).astype(np.int64)
    ordinal[ordinal == m.TERM_MISSING] = -1
    dt, dtf = sorted_rows(d_off, ordinal, d_tf, n_terms, unknown_ranks(d_keys, ordinal))
    q_off, q_terms = h.tsvector_queries(SEED, **queries)
    p_off, p_terms = pair_queries(q_off, q_terms, q_terms != m.TERM_MISSING, pair_query, len(d_off) - 1)
    return d_off.astype(np.uint32), dt, dtf, p_off, p_terms


def evaluate_pairs(m, h, pairs, sharded=False, out=None):
    """bm25x_evaluate_batch (or its sharded form) on ordinal CSR arrays.  Returns (rc, out)."""
    L = m.load_library()
    fn = L.bm25x_evaluate_batch_sharded if sharded else L.bm25x_evaluate_batch
    u32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint32)
    d_off, d_terms, d_tfs, q_off, q_terms = map(u32, pairs)
    n = len(d_off) - 1
    if out is None:
        out = np.zeros(max(n, 1), np.float64)
    p = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
    rc = fn(h, n, p(d_off, C.c_uint32), p(d_terms, C.c_uint32), p(d_tfs, C.c_uint32), p(q_off, C.c_uint32),
            p(q_terms, C.c_uint32), p(out, C.c_double))
    return rc, out


def four_step(m, h, docs, queries, pair_query=None, sharded=False):
    """Reference (b): bm25x_evaluate_batch over the four-step route."""
    rc, out = evaluate_pairs(m, h.h, four_step_pairs(m, h, docs, queries, pair_query), sharded)
    assert rc == 0, m.load_library().bm25x_last_error()
    return out[:len(docs["ent_off"]) - 1]


def evaluate_raw(m, h, docs, queries, pair_query=None, sharded=False, out=None):
    """bm25x_evaluate_tsvectors (or its sharded form) through ctypes: (rc, out); a refused call leaves out as given."""
    bm = _bm(m)
    L = m.load_library()
    keep = []
    d = bm._tsvectors(keep, **docs)
    q = bm._tsvectors(keep, **queries)
    pq = None if pair_query is None else bm._kept(keep, pair_query, np.uint32, C.c_uint32)
    if out is None:
        out = np.zeros(max(d.n, 1), np.float64)
    fn = L.bm25x_evaluate_tsvectors_sharded if sharded else L.bm25x_evaluate_tsvectors
    rc = fn(h, bm._seed(SEED), C.byref(d), C.byref(q), pq, out.ctypes.data_as(C.POINTER(C.c_double)))
    return rc, out
