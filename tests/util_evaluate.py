"""Fixtures of the bm25x_evaluate_batch tests (bm25::evaluate, crates/bm25/src/evaluate.rs:22-74), shared by the CPU and
GPU files: documents at both sides of every fieldnorm boundary, the corpus with exact lengths on which evaluate and the
search are compared, the ulp bound of that comparison, and the C call on CSR arrays."""
import ctypes as C

import numpy as np

from util_documents import documents_of_csr

U32_MAX = 0xFFFFFFFF


def fieldnorm_table(orc):
    """fieldnorm_to_length of every norm f = 0..255 (bm25.rs:278-283), as the oracle computes it."""
    return np.array([orc.lib().orc_fieldnorm_to_length(f) for f in range(256)], dtype=np.int64)


def bucket_lengths(orc):
    """Document lengths on both sides of every bucket boundary: fieldnorm_to_length(f) - 1, itself and + 1 for every f,
    then the saturation: 2^32 - 1 and sums past it.  Each as (length, tfs): the few large tfs of a document whose
    saturating Σ tf is the length (every tf >= 1, at most 2^32 - 1)."""
    out = []
    for L in fieldnorm_table(orc).tolist():
        for n in (L - 1, L, L + 1):
            if n >= 0 and all(n != x for x, _ in out):
                out.append((n, split(n)))
    out.append((U32_MAX, [U32_MAX]))
    out.append((U32_MAX, [U32_MAX - 7, 3, 5]))          # 2^32 + 1: saturates
    out.append((U32_MAX, [U32_MAX, U32_MAX, 1]))        # far past it
    return out


def split(n):
    """Up to three tfs >= 1 summing to n (none for n = 0)."""
    if n == 0:
        return []
    if n < 3:
        return [n]
    a = n // 3
    return [a, a + 1, n - 2 * a - 1] if n - 2 * a - 1 >= 1 else [n]


def sum_tf(tfs):
    """Document::length: the saturating Σ tf (vector.rs:77-83)."""
    return min(sum(int(t) for t in tfs), U32_MAX)


def exact_corpus(seed, n_docs=3000, n_terms=300, max_len=80, max_tf=20):
    """A term-major CSR whose doc_len = Σ tf, every term with postings: (n_docs, doc_len, n_terms, off, doc, tf)."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, n_terms + 1) ** 0.9
    p /= p.sum()
    rows = []
    for d in range(n_docs):
        t = np.unique(rng.choice(n_terms, size=int(rng.integers(1, max_len + 1)), p=p))
        rows.append((t, rng.integers(1, max_tf + 1, size=len(t))))
    for t in range(n_terms):                       # every term has a posting
        d = t % n_docs
        if t not in rows[d][0]:
            terms = np.append(rows[d][0], t)
            tfs = np.append(rows[d][1], 1)
            o = np.argsort(terms)
            rows[d] = (terms[o], tfs[o])
    term = np.concatenate([r[0] for r in rows]).astype(np.int64)
    tf = np.concatenate([r[1] for r in rows]).astype(np.uint32)
    doc = np.repeat(np.arange(n_docs), [len(r[0]) for r in rows])
    o = np.lexsort((doc, term))
    off = np.zeros(n_terms + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(term, minlength=n_terms))
    doc_len = np.bincount(doc, weights=tf, minlength=n_docs).astype(np.uint32)
    return n_docs, doc_len, n_terms, off, doc[o].astype(np.uint32), tf[o]


# Every term-count class of the search (1 to 64 terms, 33..64 included).
COUNTS = [1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 40, 64]


def class_queries(seed, n_terms, per_class=2):
    """per_class queries of every count of COUNTS, distinct terms ascending: (q_off u32, q_terms u32)."""
    rng = np.random.default_rng(seed)
    qs = [np.sort(rng.choice(n_terms, size=c, replace=False)) for c in COUNTS for _ in range(per_class)]
    q_off = np.zeros(len(qs) + 1, np.uint32)
    q_off[1:] = np.cumsum([len(q) for q in qs])
    return q_off, np.concatenate(qs).astype(np.uint32)


def ulp_bound(m):
    """|search - evaluate| in ulps of the larger, for a document matching m query terms.

    The search sums s0·tf / (tf + s1) with s0 = idf·(k1 + 1) rounded; evaluate sums idf·(tf·(k1 + 1) / (tf + s1)).  Both
    share idf, k1 + 1 and the rounded tf + s1; each term then takes three roundings (relative error <= 3u, u = 2^-53)
    and the ascending sum of m positive terms m - 1 more.  Each total is within (m + 2)u of the exact sum S, so the two are
    within 2(m + 2)u·S <= 2(m + 2) ulp(S) (S·u <= ulp(S)), plus one ulp for the larger of the two rounded totals."""
    return 2 * (m + 2) + 1


def ulps_apart(a, b):
    """|a - b| in ulps of max(|a|, |b|) (0 when equal)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    big = np.maximum(np.abs(a), np.abs(b))
    return np.where(a == b, 0.0, np.abs(a - b) / np.spacing(np.where(big > 0, big, 1.0)))


def search_pairs(n_docs, off, doc, tf, q_off, q_terms, rows_doc, rows_n):
    """Every (document, query) pair of the search rows, the document restated doc-major from the term-major CSR:
    (d_off, d_terms, d_tfs, p_off, p_terms, matched terms per pair, query of each pair, rank)."""
    e_off, e_term, e_tf = documents_of_csr(n_docs, off, doc, tf)
    e_off = e_off.astype(np.int64)
    qi, ids = [], []
    for i in range(len(q_off) - 1):
        n = int(rows_n[i])
        qi.extend([i] * n)
        ids.extend(rows_doc[i, :n].tolist())
    qi, ids = np.array(qi, np.int64), np.array(ids, np.int64)
    lens = e_off[ids + 1] - e_off[ids]
    d_off = np.zeros(len(ids) + 1, np.uint32)
    d_off[1:] = np.cumsum(lens)
    sel = np.concatenate([np.arange(e_off[d], e_off[d + 1]) for d in ids]) if len(ids) else np.zeros(0, np.int64)
    ql = np.diff(q_off.astype(np.int64))
    p_off = np.zeros(len(ids) + 1, np.uint32)
    p_off[1:] = np.cumsum(ql[qi])
    psel = np.concatenate([np.arange(q_off[i], q_off[i + 1]) for i in qi]) if len(qi) else np.zeros(0, np.int64)
    d_terms, p_terms = e_term[sel], q_terms[psel]
    matched = np.array([len(np.intersect1d(d_terms[d_off[p]:d_off[p + 1]], p_terms[p_off[p]:p_off[p + 1]]))
                        for p in range(len(ids))], np.int64)
    return d_off, d_terms, e_tf[sel], p_off, p_terms, matched, qi


def evaluate_csr(m, h, d_off, d_terms, d_tfs, q_off, q_terms, out=None):
    """bm25x_evaluate_batch on CSR arrays (n pairs = len(d_off) - 1).  Returns (rc, out); rc != 0 leaves out as given."""
    u32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint32)
    d_off, d_terms, d_tfs, q_off, q_terms = map(u32, (d_off, d_terms, d_tfs, q_off, q_terms))
    n = len(d_off) - 1
    if out is None:
        out = np.zeros(max(n, 1), np.float64)
    p = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
    rc = m.load_library().bm25x_evaluate_batch(h, n, p(d_off, C.c_uint32), p(d_terms, C.c_uint32), p(d_tfs, C.c_uint32),
                                               p(q_off, C.c_uint32), p(q_terms, C.c_uint32), p(out, C.c_double))
    return rc, out


def oracle_csr(oix, d_off, d_terms, d_tfs, q_off, q_terms):
    """OracleIndex.evaluate of every pair of CSR arrays."""
    return np.array([oix.evaluate(d_terms[d_off[p]:d_off[p + 1]], d_tfs[d_off[p]:d_off[p + 1]],
                                  q_terms[q_off[p]:q_off[p + 1]]) for p in range(len(d_off) - 1)], np.float64)
