"""GPU: per-query candidate lists (bm25x_search_candidates and its sharded and growing forms).

Row i of a candidate search must be, bit for bit (doc, f32, f64, payload, n), the row search_batch returns for query i
alone with allow = the bitmap of query i's candidates, and the oracle's exhaustive search with that bitmap.  Covered:
every term-count class, k from 1 to 65535, empty / single / no-term / duplicated / unsorted / complete candidate lists and
the ids 0 and n_docs - 1, ties straddling the k-th row, every source of an index handle, sharded indexes with uneven
bounds, growing segments (unsharded and sharded) with deleted ordinals and pending inserts, the refusals, concurrent
callers and the statistics."""
import ctypes as C
import threading

import numpy as np
import pytest

from util_corpora import corpus_dict
from util_cuda import D2D, cudart
from util_lib import gpu_library, refused  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import compare, live_queries, oracle_index, query_csr, same_rows

pytestmark = pytest.mark.gpu

N_DOCS = 20000
COUNTS = [1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 40, 64]   # every term-count class, 33..64 included


def bitmap(docs, n):
    b = np.zeros((n + 7) // 8, np.uint8)
    d = np.asarray(docs, np.int64)
    np.bitwise_or.at(b, d >> 3, (1 << (d & 7)).astype(np.uint8))
    return b


def cand_csr(lists):
    off = np.cumsum([0] + [len(c) for c in lists]).astype(np.uint32)
    docs = np.concatenate([np.asarray(c, np.uint32) for c in lists]) if lists else np.zeros(0, np.uint32)
    return off, docs.astype(np.uint32)


def per_query(search, q_off, q_terms, lists, k, n_ids, **kw):
    """The rows of search(q_off, q_terms, k, allow=...) run once per query with the bitmap of its candidates."""
    rows = [search(q_off[i:i + 2] - q_off[i], q_terms[q_off[i]:q_off[i + 1]], k, allow=bitmap(c, n_ids), **kw)
            for i, c in enumerate(lists)]
    out = {key: np.concatenate([r[key] for r in rows]) for key in ("doc", "score", "score64", "payload", "n")
           if rows[0].get(key) is not None}
    return out


def candidate_lists(rng, c, q_off, q_terms, n_docs):
    """One list per query, cycling through the shapes: half from documents holding a query term, half uniform; empty;
    one document; only documents holding no query term; duplicates; ids 0 and n_docs - 1; every document."""
    holders = []
    for i in range(len(q_off) - 1):
        ts = q_terms[q_off[i]:q_off[i + 1]]
        holders.append(np.unique(np.concatenate([c.post_doc[c.post_off[t]:c.post_off[t + 1]] for t in ts])))
    lists = []
    for i, h in enumerate(holders):
        shape = i % 7
        if shape == 0:
            x = np.concatenate([rng.choice(h, min(len(h), 60), replace=False), rng.integers(0, n_docs, 60)])
        elif shape == 1:
            x = np.zeros(0, np.int64)
        elif shape == 2:
            x = rng.choice(h, 1)
        elif shape == 3:
            rest = np.setdiff1d(np.arange(n_docs), h)
            x = rng.choice(rest, min(len(rest), 50), replace=False)
        elif shape == 4:
            x = np.repeat(rng.choice(h, min(len(h), 30), replace=False), 3)
        elif shape == 5:
            x = np.concatenate([[0, n_docs - 1], rng.choice(h, min(len(h), 200), replace=False), [n_docs - 1, 0]])
        else:
            x = np.arange(n_docs)
        lists.append(rng.permutation(np.asarray(x, np.int64)))   # unsorted
    return lists


@pytest.fixture(scope="module")
def world(m, orc):
    c = m.synth_corpus(0xCA4D, N_DOCS, 3000, 1, 300, 1.0)
    ix = m.Index.from_corpus(c)
    rng = np.random.default_rng(7)
    df = ix.df()
    q_off, q_terms = live_queries(rng, df, COUNTS + COUNTS)
    lists = candidate_lists(rng, c, q_off, q_terms, N_DOCS)
    yield c, ix, oracle_index(orc, c), q_off, q_terms, lists
    ix.close()


@pytest.mark.parametrize("k", [1, 10, 100, 1000, 65535])
def test_rows_equal_bitmap_search_and_oracle(m, world, k):
    c, ix, oix, q_off, q_terms, lists = world
    c_off, c_docs = cand_csr(lists)
    got = ix.search_candidates(q_off, q_terms, c_off, c_docs, k, want_payload=True)
    want = per_query(ix.search_batch, q_off, q_terms, lists, k, N_DOCS, want_payload=True)
    same_rows({key: got[key] for key in want}, want, f"k={k}")
    for i, cl in enumerate(lists):
        compare({key: got[key][i:i + 1] for key in ("doc", "score", "score64", "n")}, oix, q_off[i:i + 2] - q_off[i],
                q_terms[q_off[i]:q_off[i + 1]], k, allow=bitmap(cl, N_DOCS), what=f"k={k} q{i}")
    assert got["stats"].queries == len(q_off) - 1


def test_unknown_terms_and_empty_batch(m, world):
    c, ix, oix, q_off, q_terms, lists = world
    qs = [[c.n_terms + 5], [3, 3, 0xFFFFFFFF, 3], []]
    qo, qt = query_csr(qs)
    cl = [np.arange(100), np.arange(N_DOCS - 100, N_DOCS), np.arange(10)]
    got = ix.search_candidates(qo, qt, *cand_csr(cl), 10)
    want = per_query(ix.search_batch, qo, qt, cl, 10, N_DOCS)
    same_rows({key: got[key] for key in want}, want, "unknown terms")
    empty = ix.search_candidates(np.zeros(1, np.uint32), np.zeros(0, np.uint32), np.zeros(1, np.uint32),
                                 np.zeros(0, np.uint32), 5)
    assert empty["doc"].shape == (0, 5) and empty["stats"].queries == 0


@pytest.mark.parametrize("k", [1, 10, 137])
def test_ties_straddle_kth_row(m, orc, k):
    """One term, 400 documents of equal (tf, fieldnorm): every candidate ties with every other; the row must be the
    candidates holding the term in ascending id order."""
    rng = np.random.default_rng(11)
    n = 3000
    tie = np.sort(rng.choice(n, 400, replace=False))
    other = np.sort(rng.choice(n, 900, replace=False))
    doc_len = np.full(n, 7, np.uint32)
    kw = corpus_dict(n, [(tie, np.full(400, 2)), (other, rng.integers(1, 5, 900))], doc_len=doc_len)
    ix = m.Index(**kw)
    cand = rng.permutation(np.concatenate([rng.choice(tie, 300, replace=False), rng.integers(0, n, 200)]))
    q_off, q_terms = query_csr([[0], [0, 1]])
    got = ix.search_candidates(q_off, q_terms, *cand_csr([cand, cand]), k)
    want = per_query(ix.search_batch, q_off, q_terms, [cand, cand], k, n)
    same_rows({key: got[key] for key in want}, want, f"ties k={k}")
    held = np.intersect1d(cand, tie)
    assert np.array_equal(got["doc"][0, :min(k, len(held))], held[:k])
    oix = orc.OracleIndex(orc.Corpus(n, kw["doc_len"], 2, kw["post_off"], kw["post_doc"], kw["post_tf"]))
    compare(got, oix, q_off, q_terms, k, allow=bitmap(cand, n), what="ties")
    ix.close()


def _replica(m, src):
    rt = cudart()
    lay = src.layout()
    rep = m.Index.alloc_replica(lay, 0)
    rl = rep.layout()
    for i in range(len(rl.dev_ptr)):
        assert rt.cudaMemcpy(rl.dev_ptr[i], lay.dev_ptr[i], lay.bytes[i], D2D) == 0
    rep.finalize_replica()
    return rep


def _sealed(m, c):
    """A seal's result: the corpus's first half sealed, the rest inserted into a growing segment, then sealed."""
    h = c.n_docs // 2
    first = m.Index(h, c.doc_len[:h], c.n_terms, *_prefix_csr(c, h))
    seg = first.growing_segment()
    # the second half's documents, doc-major
    keep = c.post_doc >= h
    term = np.repeat(np.arange(c.n_terms, dtype=np.uint32), np.diff(c.post_off).astype(np.int64))[keep]
    doc, tf = c.post_doc[keep] - h, c.post_tf[keep]
    order = np.lexsort((term, doc))
    off = np.zeros(c.n_docs - h + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(doc, minlength=c.n_docs - h))
    seg.insert(off, term[order], tf[order], doc_len=c.doc_len[h:])
    out = seg.seal()[0]
    seg.close()
    first.close()
    return out


def _prefix_csr(c, h):
    term = np.repeat(np.arange(c.n_terms), np.diff(c.post_off).astype(np.int64))
    keep = c.post_doc < h
    off = np.zeros(c.n_terms + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(term[keep], minlength=c.n_terms))
    return off, c.post_doc[keep], c.post_tf[keep]


@pytest.mark.parametrize("source", ["create", "blocks_doc_len", "blocks_fieldnorm", "replica", "seal"])
def test_every_handle_source(m, world, source):
    c, ix, oix, q_off, q_terms, lists = world
    if source == "create":
        h = m.Index.from_corpus(c)
    elif source.startswith("blocks"):
        a, _ = ix.export_blocks()
        if source == "blocks_doc_len":
            a["doc_len"], a["doc_fieldnorm"], a["sum_doc_len"] = c.doc_len, None, 0
        h = m.Index.from_blocks(**a)
    elif source == "replica":
        h = _replica(m, ix)
    else:
        h = _sealed(m, c)
    n = h.info().n_docs
    cl = [np.asarray(x)[np.asarray(x) < n] for x in lists]
    for k in (10, 1000):
        got = h.search_candidates(q_off, q_terms, *cand_csr(cl), k, want_payload=True)
        want = per_query(h.search_batch, q_off, q_terms, cl, k, n, want_payload=True)
        same_rows({key: got[key] for key in want}, want, f"{source} k={k}")
    h.close()


@pytest.mark.parametrize("S", [2, 4])
def test_sharded_equals_unsharded(m, world, S):
    c, ix, oix, q_off, q_terms, lists = world
    # uneven bounds; one shard gets no candidate
    bounds, gap = ((np.array([0, 7000, N_DOCS], np.uint32), (0, 7000)) if S == 2 else
                   (np.array([0, 3000, 3100, 9000, N_DOCS], np.uint32), (3000, 3100)))
    sx = m.ShardedIndex.from_corpus(c, n_shards=S, doc_bounds=bounds)
    cl = [x[(x < gap[0]) | (x >= gap[1])] for x in lists]
    c_off, c_docs = cand_csr(cl)
    for k in (1, 10, 1000, 65535):
        got = sx.search_candidates(q_off, q_terms, c_off, c_docs, k, want_payload=True)
        want = ix.search_candidates(q_off, q_terms, c_off, c_docs, k, want_payload=True)
        same_rows({key: got[key] for key in ("doc", "score", "score64", "payload", "n")}, want, f"S={S} k={k}")
        assert got["stats"].queries == want["stats"].queries
    sx.close()


def _grow_docs(rng, n, T):
    off = np.zeros(n + 1, np.uint64)
    terms, tfs = [], []
    for d in range(n):
        t = np.sort(rng.choice(T, rng.integers(1, 12), replace=False))
        terms.append(t)
        tfs.append(rng.integers(1, 6, len(t)))
        off[d + 1] = off[d] + len(t)
    return off, np.concatenate(terms).astype(np.uint32), np.concatenate(tfs).astype(np.uint32)


@pytest.mark.parametrize("sharded", [False, True])
def test_growing_segment(m, world, sharded):
    c, ix, oix, q_off, q_terms, lists = world
    rng = np.random.default_rng(5)
    sealed = m.ShardedIndex.from_corpus(c, n_shards=3) if sharded else ix
    seg = sealed.growing_segment()
    # frequent terms so that growing documents match the queries
    T = 40
    off, term, tf = _grow_docs(rng, 300, T)
    seg.insert(off, term, tf, doc_len=np.add.reduceat(tf, off[:-1].astype(np.int64)).astype(np.uint32))
    seg.refresh()
    seg.delete(np.arange(0, 300, 7))
    off2, term2, tf2 = _grow_docs(rng, 100, T)
    seg.insert(off2, term2, tf2, doc_len=np.add.reduceat(tf2, off2[:-1].astype(np.int64)).astype(np.uint32))  # pending
    G = 400
    qs = [[0, 1], [2], [5, 9, 30], [3, 4, 6, 7, 8], list(range(10, 30))] * 2
    qo, qt = query_csr(qs)
    cl = []
    for i in range(len(qs)):
        x = np.concatenate([rng.integers(0, N_DOCS, 200), N_DOCS + rng.integers(0, G, 150), [N_DOCS + G - 1, 0]])
        cl.append(rng.permutation(x) if i % 5 else np.zeros(0, np.int64))
    for k in (1, 10, 1000):
        got = seg.search_candidates(qo, qt, *cand_csr(cl), k, want_payload=True)
        rows = []
        for i, x in enumerate(cl):
            x = np.asarray(x, np.int64)
            r = seg.search_batch(qo[i:i + 2] - qo[i], qt[qo[i]:qo[i + 1]], k, allow=bitmap(x[x < N_DOCS], N_DOCS),
                                 allow_growing=bitmap(x[x >= N_DOCS] - N_DOCS, G), allow_growing_docs=G,
                                 want_payload=True)
            rows.append(r)
        want = {key: np.concatenate([r[key] for r in rows]) for key in ("doc", "score", "score64", "payload", "n")}
        same_rows({key: got[key] for key in want}, want, f"growing sharded={sharded} k={k}")
        d = got["doc"][got["doc"] != 0xFFFFFFFF].astype(np.int64)
        assert not np.isin(d - N_DOCS, np.arange(0, 300, 7)).any(), "a deleted ordinal came back"
    assert seg.info().pending == 0
    code, msg = refused(m, lambda: seg.search_candidates(qo[:2], qt[:qo[1]], *cand_csr([[N_DOCS + G]]), 10))
    assert code == 1 and "query 0" in msg and f"doc id {N_DOCS + G}" in msg
    seg.close()
    if sharded:
        sealed.close()


def _raw_call(m, fn, h, q_off, q_terms, c_off, c_docs, k):
    """The call through ctypes on output buffers filled with a pattern: (status, message, outputs untouched)."""
    L = m.load_library()
    nq = len(q_off if q_off is not None else c_off) - 1
    kk = max(k, 1)
    outs = [np.full(nq * kk, 0xAB, np.uint32), np.full(nq * kk, 7.0, np.float32), np.full(nq * kk, 7.0),
            np.full(nq * kk * 3, 0xAB, np.uint16), np.full(nq, 0xAB, np.uint32)]
    pattern = [o.copy() for o in outs]
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t)) if a is not None else None
    q_off = None if q_off is None else np.ascontiguousarray(q_off, np.uint32)
    c_off = None if c_off is None else np.ascontiguousarray(c_off, np.uint32)
    rc = getattr(L, fn)(h, nq, P(q_off, C.c_uint32), P(np.ascontiguousarray(q_terms, np.uint32), C.c_uint32),
                        P(c_off, C.c_uint32), None if c_docs is None else P(np.ascontiguousarray(c_docs, np.uint32), C.c_uint32), k,
                        P(outs[0], C.c_uint32), P(outs[1], C.c_float), P(outs[2], C.c_double), P(outs[3], C.c_uint16),
                        P(outs[4], C.c_uint32), None)
    msg = L.bm25x_last_error().decode() if rc else ""
    return rc, msg, all(np.array_equal(a, b) for a, b in zip(outs, pattern))


def test_refusals(m, world):
    c, ix, oix, q_off, q_terms, lists = world
    q1 = np.array([0, 2], np.uint32)
    t1 = np.array([1, 2], np.uint32)
    c1 = np.array([0, 3], np.uint32)
    d1 = np.array([5, 6, 7], np.uint32)
    df = ix.df()
    live65 = np.flatnonzero(df > 0)[:65].astype(np.uint32)
    rep = m.Index.alloc_replica(ix.layout(), 0)
    sx = m.ShardedIndex.from_corpus(c, n_shards=2)
    cases = [
        ("null index", None, q1, t1, c1, d1, 10, 1, "null argument"),
        ("null q_off", ix.h, None, t1, c1, d1, 10, 1, "null argument"),
        ("null c_off", ix.h, q1, t1, None, d1, 10, 1, "null argument"),
        ("k == 0", ix.h, q1, t1, c1, d1, 0, 5, "number of needed rows is set to 0"),
        ("k > max", ix.h, q1, t1, c1, d1, 65536, 4, "BM25X_MAX_K"),
        ("q_off", ix.h, np.array([0, 2, 1], np.uint32), t1, np.array([0, 3, 3], np.uint32), d1, 10, 1, "q_off not monotone at 1"),
        ("65 live terms", ix.h, np.array([0, 65], np.uint32), live65, c1[:2], d1, 10, 4, "65 live terms"),
        ("c_off", ix.h, np.array([0, 1, 2], np.uint32), t1, np.array([0, 3, 1], np.uint32), d1, 10, 1, "c_off not monotone at 1"),
        # a later offset going backwards is refused before an earlier, huge one leads the id check past the list
        ("c_off past the list", ix.h, np.array([0, 1, 2], np.uint32), t1, np.array([0, 1_000_000_000, 5], np.uint32),
         np.arange(5, dtype=np.uint32), 10, 1, "c_off not monotone at 1"),
        ("c_off with null c_docs", ix.h, np.array([0, 1, 2], np.uint32), t1, np.array([0, 3, 0], np.uint32), None, 10, 1,
         "c_off not monotone at 1"),
        ("candidate id", ix.h, q1, t1, c1, np.array([5, N_DOCS, 7], np.uint32), 10, 1,
         f"query 0, candidate entry 1: doc id {N_DOCS}"),
        ("replica", rep.h, q1, t1, c1, d1, 10, 1, "not finalized"),
    ]
    for what, h, qo, qt, co, cd, k, code, text in cases:
        rc, msg, untouched = _raw_call(m, "bm25x_search_candidates", h, qo, qt, co, cd, k)
        assert rc == code and text in msg, (what, rc, msg)
        assert untouched, f"{what}: a refused call wrote output"
    # the sharded form: the whole segment's canonicalisation, then the candidates against the whole segment's ids
    for what, qo, qt, co, cd, code, text in [
            ("sharded 65 live terms", np.array([0, 65], np.uint32), live65, c1[:2], d1, 4, "65 live terms"),
            ("sharded candidate id", q1, t1, c1, np.array([5, 6, N_DOCS + 3], np.uint32), 1, f"doc id {N_DOCS + 3}")]:
        rc, msg, untouched = _raw_call(m, "bm25x_search_candidates_sharded", sx.h, qo, qt, co, cd, 10)
        assert rc == code and text in msg and untouched, (what, rc, msg)
    rep.close()
    sx.close()


def test_concurrent_callers(m, world):
    c, ix, oix, q_off, q_terms, lists = world
    c_off, c_docs = cand_csr(lists)
    want_c = ix.search_candidates(q_off, q_terms, c_off, c_docs, 10)
    want_b = ix.search_batch(q_off, q_terms, 10)
    errors = []

    def run(fn, want, what):
        try:
            for _ in range(6):
                same_rows({key: v for key, v in fn().items() if key in want}, {k: v for k, v in want.items() if k != "stats"},
                          what)
        except BaseException as e:   # reported by the main thread
            errors.append(e)

    ts = [threading.Thread(target=run, args=(lambda: ix.search_candidates(q_off, q_terms, c_off, c_docs, 10), want_c,
                                             f"candidates {i}")) for i in range(2)]
    ts.append(threading.Thread(target=run, args=(lambda: ix.search_batch(q_off, q_terms, 10), want_b, "batch")))
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[0]


def test_stats(m, world):
    c, ix, oix, q_off, q_terms, lists = world
    got = ix.search_candidates(q_off, q_terms, *cand_csr(lists), 10)
    st = got["stats"]
    df = ix.df().astype(np.uint64)
    assert st.queries == len(q_off) - 1
    assert st.launches == 4
    assert st.kernel_ms > 0
    assert st.postings == int(df[q_terms].sum())
    assert st.postings_fetched > 0
    none = ix.search_candidates(q_off, q_terms, np.zeros(len(q_off), np.uint32), np.zeros(0, np.uint32), 10)
    assert none["stats"].launches == 0 and np.all(none["n"] == 0) and np.all(none["doc"] == 0xFFFFFFFF)
