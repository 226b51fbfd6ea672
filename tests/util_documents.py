"""Documents as bm25x_index_create_from_documents takes them, and the numpy restatement of the reference's Segment of
those documents (crates/bm25/src/io.rs:187-244: Record(length, payload) per document in input order, Mapping(key, doc,
tf) per element sorted by (key, doc)): the CSR bm25x_index_create builds the handle a build from documents must equal."""
from types import SimpleNamespace

import numpy as np
import scipy.sparse


def documents_of_csr(n_docs, post_off, post_doc, post_tf):
    """A term-major CSR transposed to documents: (elem_off u64, elem_term u32, elem_tf u32), terms ascending inside each
    document (scipy's transposition keeps the column order)."""
    T = len(post_off) - 1
    m = scipy.sparse.csc_matrix((np.asarray(post_tf, np.uint32), np.asarray(post_doc), np.asarray(post_off, np.int64)),
                                shape=(int(n_docs), T)).tocsr()
    return m.indptr.astype(np.uint64), m.indices.astype(np.uint32), m.data.astype(np.uint32)


def key_words(keys):
    """[n, 16] keys as (hi, lo) big-endian u64 words: their order is the bytewise order of the keys."""
    k = np.ascontiguousarray(keys, dtype=np.uint8).reshape(-1, 16)
    w = k.view(">u8").reshape(-1, 2)
    return w[:, 0].astype(np.uint64), w[:, 1].astype(np.uint64)


def vocabulary(elem_key):
    """The distinct keys ascending bytewise ([T, 16] u8) and each element's ordinal among them."""
    hi, lo = key_words(elem_key)
    order = np.lexsort((lo, hi))
    if len(order) == 0:
        return np.zeros((0, 16), np.uint8), np.zeros(0, np.uint32)
    h, l = hi[order], lo[order]
    first = np.ones(len(order), bool)
    first[1:] = (h[1:] != h[:-1]) | (l[1:] != l[:-1])
    rank = np.cumsum(first) - 1
    ordinal = np.empty(len(order), np.uint32)
    ordinal[order] = rank
    keys = np.ascontiguousarray(elem_key, dtype=np.uint8).reshape(-1, 16)[order[first]]
    return keys, ordinal


def segment(elem_off, elem_tf, elem_term=None, elem_key=None, n_terms=0):
    """The Segment of the documents as a CSR (namespace: n_docs, doc_len, n_terms, post_off, post_doc, post_tf, term_keys):
    doc_len = the saturating Σ tf of each document (Document::length, vector.rs:76-83), the mappings stable-sorted by term
    (they arrive in doc order), keyed: the terms are the distinct keys ascending."""
    off = np.asarray(elem_off, np.int64)
    N = len(off) - 1
    tf = np.asarray(elem_tf, np.uint32)
    keys = None
    if elem_key is not None:
        keys, term = vocabulary(elem_key)
        T = len(keys)
    else:
        term, T = np.asarray(elem_term, np.uint32), int(n_terms)
    doc = np.repeat(np.arange(N, dtype=np.uint32), np.diff(off))
    sums = np.zeros(N, np.uint64)
    np.add.at(sums, doc, tf.astype(np.uint64))
    order = np.argsort(term, kind="stable")
    post_off = np.zeros(T + 1, np.uint64)
    post_off[1:] = np.cumsum(np.bincount(term, minlength=T))
    return SimpleNamespace(n_docs=N, doc_len=np.minimum(sums, 0xFFFFFFFF).astype(np.uint32), n_terms=T, post_off=post_off,
                           post_doc=doc[order], post_tf=tf[order], term_keys=keys)


CHUNK = 1 << 22  # elements per chunk of the device build (bm25x_documents.cu)


def vocab_schedule(elem_key):
    """The restated loop of vocab_pass over keyed elements: one event per chunk c, in order, ("grow", c, capacity,
    kept) when the list is reallocated keeping its first `kept` entries, then ("defer", c, A) or ("compact", c, A) with
    A the appended entries the chunk leaves.  A compaction leaves V = the distinct keys of every element so far, counted
    from each key's first occurrence."""
    E = len(elem_key)
    _, ordinal = vocabulary(elem_key)
    first = np.full(int(ordinal.max()) + 1 if E else 0, E, np.int64)
    np.minimum.at(first, ordinal, np.arange(E, dtype=np.int64))
    first.sort()
    events, V, A, cap = [], 0, 0, 0
    for c, g in enumerate(range(0, E, CHUNK)):
        n = min(CHUNK, E - g)
        if V + A + n > cap:
            cap = 2 * (V + A + n)
            events.append(("grow", c, cap, V + A))
        A += n
        if A >= max(V, CHUNK) or g + n == E:
            events.append(("compact", c, A))
            V, A = int(np.searchsorted(first, g + n)), 0
        else:
            events.append(("defer", c, A))
    return events


def csr_kwargs(s):
    """A segment() namespace as the keyword arguments of Index / ShardedIndex."""
    return dict(n_docs=s.n_docs, doc_len=s.doc_len, n_terms=s.n_terms, post_off=s.post_off, post_doc=s.post_doc,
                post_tf=s.post_tf, term_keys=s.term_keys)
