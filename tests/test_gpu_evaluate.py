"""GPU: bm25x_evaluate_batch (k_evaluate, bm25::evaluate behind `<&>` without an index scan) against the oracle's evaluate
over the same corpus and statistics, bit for bit:
- documents at both sides of every fieldnorm boundary and past the saturation of Σ tf, at four (k1, b);
- every kind of handle: bm25x_index_create, stored blocks in both norm forms, documents keyless and keyed, tsvectors, a
  finalized replica, and that replica refilled from a corpus with other df and finalized again; a growing handle and a
  replica of one are refused and write nothing;
- queries of 9 to 5 000 terms mixed with unknown ordinals, BM25X_TERM_MISSING and df-0 terms, a document of 10^6
  elements, empty documents and queries, and one call of more than 2·10^6 pairs;
- agreement with the search within the ulp bound of tests/util_evaluate.py on every row at k = 1000;
- tsvector documents cast on the GPU, their unknown lexemes numbered past the vocabulary;
- eight threads on a fresh handle, and device memory across repeated calls and refusals."""
import threading

import numpy as np
import pytest

from oracle.oracle import EncodedBlocks
from util_cuda import D2D, cudart, free_bytes
from util_documents import documents_of_csr, segment, vocabulary
from util_evaluate import (COUNTS, U32_MAX, bucket_lengths, class_queries, evaluate_csr, exact_corpus, oracle_csr,
                           search_pairs, ulp_bound, ulps_apart)
from util_index import fieldnorms
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_segment import random_keys
from util_tsvector import pack, synthetic

pytestmark = pytest.mark.gpu

N_EMPTY = 4    # terms past the corpus's last with no postings (df 0)
SEED = bytes(range(32))


class World:
    """An exact-length corpus of T terms with postings and N_EMPTY more without, its oracle and its create handle."""

    def __init__(self, m, orc, seed, k1=1.2, b=0.75, n_docs=2000, n_terms=200):
        n, dl, T, off, doc, tf = exact_corpus(seed, n_docs=n_docs, n_terms=n_terms)
        self.n, self.dl, self.T, self.doc, self.tf, self.k1, self.b = n, dl, T + N_EMPTY, doc, tf, k1, b
        self.off = np.concatenate([off, np.full(N_EMPTY, off[-1], np.uint64)])
        self.corpus = orc.Corpus(n, dl, self.T, self.off, doc, tf, k1, b)
        self.oix = orc.OracleIndex(self.corpus)
        self.ix = m.Index(n, dl, self.T, self.off, doc, tf, k1=k1, b=b)

    def close(self):
        self.ix.close()


def csr(rows):
    """(off u32, flat u32) of a list of arrays."""
    off = np.zeros(len(rows) + 1, np.uint32)
    off[1:] = np.cumsum([len(r) for r in rows])
    flat = np.concatenate([np.asarray(r, np.uint32) for r in rows]) if rows else np.zeros(0, np.uint32)
    return off, flat.astype(np.uint32)


def random_pairs(rng, n, vocab, max_d=40, max_q=12, max_tf=50, missing=True):
    """n (document, query) pairs over ordinals < vocab, TERM_MISSING closing every third query: (d_off, d_terms, d_tfs,
    q_off, q_terms)."""
    dt, dtf, qt = [], [], []
    for i in range(n):
        d = np.sort(rng.choice(vocab, size=int(rng.integers(0, max_d + 1)), replace=False))
        q = set(rng.choice(vocab, size=int(rng.integers(0, max_q + 1)), replace=False).tolist())
        if len(d):   # share some of the document's terms
            q |= set(rng.choice(d, size=int(rng.integers(0, len(d) + 1)), replace=False).tolist())
        q = sorted(q) + ([U32_MAX] if missing and i % 3 == 0 else [])
        dt.append(d)
        dtf.append(rng.integers(1, max_tf + 1, size=len(d)))
        qt.append(q)
    d_off, d_terms = csr(dt)
    _, d_tfs = csr(dtf)
    q_off, q_terms = csr(qt)
    return d_off, d_terms, d_tfs, q_off, q_terms


def check(m, h, oix, pairs, what):
    rc, got = evaluate_csr(m, h, *pairs)
    assert rc == 0, (what, m.load_library().bm25x_last_error())
    want = oracle_csr(oix, *pairs)
    n = len(pairs[0]) - 1
    assert np.array_equal(got[:n], want), (what, np.flatnonzero(got[:n] != want)[:10])
    return want


K1_B = [(1.2, 0.75), (1.2, 0.0), (2.0, 1.0), (2.0, 0.75)]


@pytest.mark.parametrize("k1,b", K1_B)
def test_every_fieldnorm_bucket(m, orc, k1, b):
    """Documents of length fieldnorm_to_length(f) - 1, itself and + 1 for every f, and of 2^32 - 1 and more (saturated),
    each of up to three elements with large tf, against a query of its terms and one of its first term."""
    w = World(m, orc, 21, k1, b)
    rng = np.random.default_rng(22)
    dt, dtf, qt = [], [], []
    for n, tfs in bucket_lengths(orc):
        t = np.sort(rng.choice(w.T, size=len(tfs), replace=False))
        for q in (t, t[:1]):
            dt.append(t)
            dtf.append(tfs)
            qt.append(np.union1d(q, rng.choice(w.T + 10, size=2, replace=False)))
    d_off, d_terms = csr(dt)
    _, d_tfs = csr(dtf)
    q_off, q_terms = csr(qt)
    want = check(m, w.ix.h, w.oix, (d_off, d_terms, d_tfs, q_off, q_terms), f"k1={k1} b={b}")
    assert np.count_nonzero(want) > len(want) * 0.8
    w.close()


def _replica(m, src):
    lay = src.layout()
    rep = m.Index.alloc_replica(lay, 0)
    rl = rep.layout()
    for i in range(len(rl.dev_ptr)):
        assert cudart().cudaMemcpy(rl.dev_ptr[i], lay.dev_ptr[i], lay.bytes[i], D2D) == 0
    rep.finalize_replica()
    return rep


def _blocks(m, orc, w, **kw):
    eb = EncodedBlocks(orc.Corpus(w.n, w.dl, w.T, w.off, w.doc, w.tf))
    return m.Index.from_blocks(w.n, w.T, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf, eb.doc_off,
                               eb.tf_off, eb.bytes[:eb.n_bytes], k1=w.k1, b=w.b, **kw)


KINDS = ["create", "blocks-doc_len", "blocks-fieldnorm", "documents-keyless", "documents-keyed", "replica"]


@pytest.mark.parametrize("kind", KINDS)
def test_handle_kinds(m, orc, kind):
    """Each kind of handle over one corpus (k1 = 1.6, b = 0.6) against the oracle.  The stored-norm blocks have no exact
    lengths; with the caller's Σlen equal to the corpus's they score with its statistics, and equal the create handle."""
    w = World(m, orc, 31, 1.6, 0.6)
    rng = np.random.default_rng(32)
    pairs = random_pairs(rng, 800, w.T + 40)
    e_off, e_term, e_tf = documents_of_csr(w.n, w.off, w.doc, w.tf)
    if kind == "create":
        h = w.ix
    elif kind == "blocks-doc_len":
        h = _blocks(m, orc, w, doc_len=w.dl)
    elif kind == "blocks-fieldnorm":
        h = _blocks(m, orc, w, doc_fieldnorm=fieldnorms(orc, w.dl), sum_doc_len=int(w.dl.astype(np.uint64).sum()))
    elif kind == "documents-keyless":
        h = m.Index.from_documents(e_off, e_tf, elem_term=e_term, n_terms=w.T, k1=w.k1, b=w.b)
    elif kind == "documents-keyed":
        # keys ascending with the ordinals: the vocabulary (the distinct keys of the elements) numbers the terms with
        # postings as the corpus does and drops the df-0 ones, which evaluate skips either way
        keys = np.array(sorted(random_keys(rng, w.T).tolist()), np.uint8)
        h = m.Index.from_documents(e_off, e_tf, elem_key=keys[e_term], k1=w.k1, b=w.b)
        assert h.info().n_terms == w.T - N_EMPTY
    else:
        h = _replica(m, w.ix)
    want = check(m, h.h, w.oix, pairs, kind)
    assert np.count_nonzero(want) > 300
    if h is not w.ix:
        rc, same = evaluate_csr(m, w.ix.h, *pairs)
        assert rc == 0 and np.array_equal(same[:len(want)], want)
        h.close()
    w.close()


def _same_shape_other_df(rng, w):
    """A corpus with the replica's layout (N, T, padded list lengths and block counts) and other df: one more posting in
    every list whose padded length and block count that keeps.  Exact lengths."""
    df = np.diff(w.off.astype(np.int64))
    grow = (df % 4 != 0) & (df % 128 != 0) & (df < w.n)
    lists = [np.sort(rng.choice(w.n, size=int(n), replace=False)) for n in df + grow]
    off = np.zeros(w.T + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in lists])
    doc = np.concatenate(lists).astype(np.uint32)
    tf = rng.integers(1, 20, size=len(doc)).astype(np.uint32)
    dl = np.maximum(np.bincount(doc, weights=tf, minlength=w.n), 1).astype(np.uint32)
    return grow, off, doc, tf, dl


def test_replica_refilled_scores_with_the_new_df(m, orc):
    """A replica evaluated (its idf table built), refilled from a corpus of the same layout with other df and finalized
    again: evaluate scores with the new corpus's df, as an index built from it does."""
    w = World(m, orc, 41)
    rng = np.random.default_rng(42)
    pairs = random_pairs(rng, 800, w.T + 20)
    rep = _replica(m, w.ix)
    first = check(m, rep.h, w.oix, pairs, "replica")
    grow, off, doc, tf, dl = _same_shape_other_df(rng, w)
    assert grow.sum() > 50
    ix2 = m.Index(w.n, dl, w.T, off, doc, tf)
    lay, rl = ix2.layout(), rep.layout()
    for i in range(len(rl.dev_ptr)):
        assert rl.bytes[i] == lay.bytes[i]
        assert cudart().cudaMemcpy(rl.dev_ptr[i], lay.dev_ptr[i], lay.bytes[i], D2D) == 0
    rep.finalize_replica()
    assert np.array_equal(rep.df(), np.diff(off.astype(np.int64)).astype(np.uint32))
    oix2 = orc.OracleIndex(orc.Corpus(w.n, dl, w.T, off, doc, tf))
    second = check(m, rep.h, oix2, pairs, "replica refilled")
    assert np.count_nonzero(second != first) > 100
    rc, built = evaluate_csr(m, ix2.h, *pairs)
    assert rc == 0 and np.array_equal(built[:len(second)], second)
    rep.close()
    ix2.close()
    w.close()


def _refused(m, h, pairs, what, msg):
    n = len(pairs[0]) - 1
    out = np.full(n, np.nan).view(np.uint64)
    out[:] = 0x7FF4DEADBEEF0000 + np.arange(n, dtype=np.uint64)
    before = out.copy()
    rc, _ = evaluate_csr(m, h, *pairs, out=out.view(np.float64))
    assert rc == 1 and msg in m.load_library().bm25x_last_error().decode(), what
    assert np.array_equal(out, before), f"{what}: a refused call wrote its output"


def test_growing_handle_refused(m, orc):
    """bm25x_growing_create's handle scores with the sealed segment's avgdl but holds the growing documents' N and df:
    evaluate refuses it, and a replica of it, as the export does, and writes nothing."""
    w = World(m, orc, 51)
    rng = np.random.default_rng(52)
    g_off, g_term, g_tf = [0], [], []
    for _ in range(300):
        t = np.sort(rng.choice(w.T, size=int(rng.integers(1, 10)), replace=False))
        g_term.extend(t.tolist())
        g_tf.extend(rng.integers(1, 4, size=len(t)).tolist())
        g_off.append(len(g_term))
    g_len = np.bincount(np.repeat(np.arange(300), np.diff(g_off)), weights=g_tf, minlength=300).astype(np.uint32)
    g = w.ix.growing(np.array(g_off, np.uint64), np.array(g_term, np.uint32), np.array(g_tf, np.uint32), doc_len=g_len)
    assert g.info().avgdl == w.ix.info().avgdl != g_len.sum() / 300
    pairs = random_pairs(rng, 50, w.T)
    msg = "another segment's statistics"
    _refused(m, g.h, pairs, "growing handle", msg)
    with pytest.raises(m.Bm25xError) as e:
        g.export_blocks()
    assert e.value.code == 1 and msg in str(e.value)
    rep = _replica(m, g)
    _refused(m, rep.h, pairs, "replica of a growing handle", msg)
    # the sealed index it scores with still evaluates
    check(m, w.ix.h, w.oix, pairs, "sealed index")
    rep.close()
    g.close()
    w.close()


def test_query_and_document_shapes(m, orc):
    """Queries of 9, 33, 64, 65 and 5 000 terms (known, df 0, ordinals >= n_terms, TERM_MISSING), a document of 10^6
    elements, empty documents and empty queries."""
    w = World(m, orc, 61)
    rng = np.random.default_rng(62)
    big = np.sort(rng.choice(2_000_000, size=1_000_000, replace=False))
    big = np.union1d(big, np.arange(w.T)).astype(np.uint32)[:1_000_000]
    big_tf = rng.integers(1, 1000, size=len(big)).astype(np.uint32)
    assert len(big) == 1_000_000 and big[w.T - 1] == w.T - 1
    docs = [(np.zeros(0, np.uint32), np.zeros(0, np.uint32)), (big, big_tf)]
    for _ in range(6):
        t = np.sort(rng.choice(w.T + 6000, size=int(rng.integers(1, 3000)), replace=False))
        docs.append((t, rng.integers(1, 30, size=len(t))))
    queries = [np.zeros(0, np.uint32)]
    for n in (9, 33, 64, 65, 5000):
        known = rng.choice(w.T - N_EMPTY, size=min(n // 2, w.T - N_EMPTY), replace=False)
        empty = np.arange(w.T - N_EMPTY, w.T)[:max(1, n // 10)]
        rest = rng.choice(np.arange(w.T, w.T + 20_000), size=n, replace=False)
        q = np.union1d(np.union1d(known, empty), rest)[:n - 1]
        queries.append(np.append(np.sort(q), U32_MAX))
        assert len(queries[-1]) == n and len(np.unique(queries[-1])) == n
    dt, dtf, qt = [], [], []
    for d in docs:
        for q in queries:
            dt.append(d[0])
            dtf.append(d[1])
            qt.append(q)
    d_off, d_terms = csr(dt)
    _, d_tfs = csr(dtf)
    q_off, q_terms = csr(qt)
    want = check(m, w.ix.h, w.oix, (d_off, d_terms, d_tfs, q_off, q_terms), "shapes")
    nq = len(queries)
    assert np.all(want[:nq] == 0) and np.all(want[::nq] == 0)         # empty document, empty query
    assert np.all(want[nq + 1:2 * nq] > 0)                              # the 10^6-element document
    w.close()


def test_two_million_pairs_in_one_call(m, orc):
    """One call of 2 048 000 pairs (16 000 blocks of 128 threads): 2 048 distinct pairs repeated 1 000 times, each
    against the oracle."""
    w = World(m, orc, 71)
    rng = np.random.default_rng(72)
    base = random_pairs(rng, 2048, w.T + 20, max_d=12, max_q=6)
    want = oracle_csr(w.oix, *base)
    reps = 1000
    d_off, d_terms, d_tfs, q_off, q_terms = base

    def tile(off, flat):
        lens = np.tile(np.diff(off.astype(np.int64)), reps)
        o = np.zeros(len(lens) + 1, np.uint32)
        o[1:] = np.cumsum(lens)
        return o, np.tile(flat, reps)

    big_d_off, big_d_terms = tile(d_off, d_terms)
    _, big_d_tfs = tile(d_off, d_tfs)
    big_q_off, big_q_terms = tile(q_off, q_terms)
    rc, got = evaluate_csr(m, w.ix.h, big_d_off, big_d_terms, big_d_tfs, big_q_off, big_q_terms)
    assert rc == 0 and len(got) == 2048 * reps >= 2_000_000
    assert np.array_equal(got, np.tile(want, reps))
    assert np.count_nonzero(want) > 500
    w.close()


def test_agreement_with_the_search(m, orc):
    """Every row of search_batch at k = 1000 for two queries of every term-count class, evaluated with the document restated
    doc-major: within ulp_bound of the row's f64 score, and equal to the oracle's evaluate."""
    n, dl, T, off, doc, tf = exact_corpus(5)                    # the fixture of tests/test_evaluate.py
    ix = m.Index(n, dl, T, off, doc, tf)
    oix = orc.OracleIndex(orc.Corpus(n, dl, T, off, doc, tf))
    q_off, q_terms = class_queries(6, T)
    res = ix.search_batch(q_off, q_terms, 1000)
    assert np.count_nonzero(res["n"] == 1000) >= len(COUNTS)
    d_off, d_terms, d_tfs, p_off, p_terms, matched, qi = search_pairs(n, off, doc, tf, q_off, q_terms, res["doc"],
                                                                    res["n"])
    rc, got = evaluate_csr(m, ix.h, d_off, d_terms, d_tfs, p_off, p_terms)
    assert rc == 0
    score = np.concatenate([res["score64"][i, :res["n"][i]] for i in range(len(q_off) - 1)])
    apart = ulps_apart(got, score)
    assert np.all(apart <= np.array([ulp_bound(int(x)) for x in matched]))
    assert np.array_equal(got, oracle_csr(oix, d_off, d_terms, d_tfs, p_off, p_terms))
    ix.close()


def test_tsvector_index_and_tsvector_documents(m, orc):
    """An index from tsvectors against the oracle over the restated segment, evaluated on tsvector documents cast on the
    GPU: known keys take their ordinals (lookup_terms), unknown keys distinct ordinals >= n_terms in key order, each
    document re-sorted by ordinal.  Its length counts the unknown lexemes (Document::length)."""
    rng = np.random.default_rng(81)
    tsv, words, _ = synthetic(rng, 600, 5, 40, 800, 0.2)
    ix = m.Index.from_tsvectors(SEED, **tsv, k1=1.4, b=0.7)
    off, keys, tf = m.cast_tsvectors(SEED, **tsv)
    s = segment(off, tf, elem_key=keys)
    assert ix.info().n_terms == s.n_terms
    oix = orc.OracleIndex(orc.Corpus(s.n_docs, s.doc_len, s.n_terms, s.post_off, s.post_doc, s.post_tf, 1.4, 0.7))
    # documents: lexemes of the index's words and new ones, some repeated inside a vector (the cast merges them)
    new = [bytes(rng.integers(97, 123, size=int(rng.integers(1, 30)), dtype=np.uint8)) + b"#" for _ in range(200)]
    vec_lens, lex, npos = [], [], []
    for i in range(300):
        n_old, n_new = int(rng.integers(0, 30)), int(rng.integers(0, 6)) if i % 4 else 0
        pick = [words[j] for j in rng.integers(0, len(words), n_old)] + [new[j] for j in rng.integers(0, 200, n_new)]
        vec_lens.append(len(pick))
        lex.extend(pick)
        npos.extend(int(rng.integers(1, 5)) for _ in pick)      # the document cast wants positions (tsvector.rs:88)
    docs = pack(vec_lens, lex, npos)
    d_off, d_keys, d_tf = m.cast_tsvectors(SEED, **docs)
    ordinal = ix.lookup_terms(d_keys).astype(np.int64)
    unknown = ordinal == m.TERM_MISSING
    _, rank = vocabulary(d_keys[unknown])
    ordinal[unknown] = s.n_terms + rank.astype(np.int64)
    dt, dtf, qt, lens, has_new = [], [], [], [], []
    for i in range(len(d_off) - 1):
        a, b = int(d_off[i]), int(d_off[i + 1])
        o = np.argsort(ordinal[a:b])
        dt.append(ordinal[a:b][o])
        dtf.append(d_tf[a:b][o])
        doc_i = m.Document(dt[-1], dtf[-1])
        lens.append(doc_i.length())
        has_new.append(bool(unknown[a:b].any()))
        q = np.union1d(rng.choice(dt[-1], size=min(len(dt[-1]), 5), replace=False) if len(dt[-1]) else [],
                       rng.choice(s.n_terms + 10, size=3, replace=False))
        qt.append(q.astype(np.uint32))
    assert lens == [int(min(int(d_tf[int(d_off[i]):int(d_off[i + 1])].astype(np.uint64).sum()), U32_MAX))
                    for i in range(len(d_off) - 1)]
    assert sum(has_new) > 100
    p_doff, p_dt = csr(dt)
    _, p_dtf = csr(dtf)
    p_qoff, p_qt = csr(qt)
    want = check(m, ix.h, oix, (p_doff, p_dt, p_dtf, p_qoff, p_qt), "tsvector documents")
    # the unknown lexemes count in the length: without them the documents score otherwise
    known_only = [(t[t < s.n_terms], f[t < s.n_terms]) for t, f in zip(dt, dtf)]
    k_off, k_dt = csr([x[0] for x in known_only])
    _, k_dtf = csr([x[1] for x in known_only])
    rc, without = evaluate_csr(m, ix.h, k_off, k_dt, k_dtf, p_qoff, p_qt)
    assert rc == 0
    changed = (without[:len(want)] != want) & (want > 0)
    assert np.count_nonzero(changed & np.array(has_new)) > 30 and not np.any(changed & ~np.array(has_new))
    ix.close()


def test_concurrent_first_use_and_memory(m, orc):
    """Eight threads on a fresh handle whose evaluate tables are not built yet, each calling evaluate and search_batch:
    every result equals a serial run.  Refused calls write nothing, and after the first call device memory is unchanged
    across repeated calls and refusals."""
    w = World(m, orc, 91)
    rng = np.random.default_rng(92)
    pairs = [random_pairs(rng, 400, w.T + 20) for _ in range(8)]
    q_off, q_terms = class_queries(93, w.T - N_EMPTY, per_class=1)
    got = [None] * 8
    gate = threading.Barrier(8)

    def run(i):
        gate.wait()
        rc, ev = evaluate_csr(m, w.ix.h, *pairs[i])
        res = w.ix.search_batch(q_off, q_terms, 10)
        got[i] = (rc, ev, res)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for i in range(8):
        rc, ev, res = got[i]
        assert rc == 0
        rc2, ev2 = evaluate_csr(m, w.ix.h, *pairs[i])
        assert rc2 == 0 and np.array_equal(ev, ev2), i
        assert np.array_equal(ev[:len(pairs[i][0]) - 1], oracle_csr(w.oix, *pairs[i])), i
        serial = w.ix.search_batch(q_off, q_terms, 10)
        for key in ("doc", "score64", "n"):
            assert np.array_equal(res[key], serial[key]), (i, key)
    before = free_bytes()
    d_off, d_terms, d_tfs, q_off2, q_terms2 = pairs[0]
    bad_tf = d_tfs.copy()
    bad_tf[len(bad_tf) // 2] = 0
    bad_q = q_terms2.copy()
    j = int(np.flatnonzero(np.diff(q_off2.astype(np.int64)) >= 2)[0])
    bad_q[q_off2[j]], bad_q[q_off2[j] + 1] = bad_q[q_off2[j] + 1], bad_q[q_off2[j]]
    for _ in range(3):
        rc, _ = evaluate_csr(m, w.ix.h, *pairs[1])
        assert rc == 0
        _refused(m, w.ix.h, (d_off, d_terms, bad_tf, q_off2, q_terms2), "tf = 0", "zero term frequency")
        _refused(m, w.ix.h, (d_off, d_terms, d_tfs, q_off2, bad_q), "descending query", "not strictly ascending")
        _refused(m, w.ix.h, (d_off, d_terms, None, q_off2, q_terms2), "no tfs", "null argument")
    assert free_bytes() == before
    w.close()
