"""GPU: indexes built from documents (bm25x_index_create_from_documents, bm25x_index_create_sharded_from_documents)
against bm25x_index_create / bm25x_sharded_create on the numpy restatement of the reference's Segment of the same
documents (tests/util_documents.py): every array the handle reports, its info and df, search rows (and the oracle's), the
golden passages' rankings, and the stored blocks a keyed handle exports."""
import numpy as np
import pytest

from util_cuda import free_bytes
from util_documents import csr_kwargs, documents_of_csr, key_words, segment
from util_index import DERIVED, LAYOUT, SCALARS, check_shards, read_back
from util_lib import gpu_library, refused  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import compare, oracle_index, query_csr, same_rows

pytestmark = pytest.mark.gpu

CHUNK = 1 << 22  # elements per chunk of the device build (bm25x_documents.cu)


def _same_arrays(lg, dg, lw, dw, what):
    """Two handles' layout and derived arrays byte-identical (placeholder slots of empty arrays aside)."""
    for name in SCALARS:
        assert getattr(lg, name) == getattr(lw, name), f"{what}: {name} {getattr(lg, name)} != {getattr(lw, name)}"
    assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min, what
    ag, aw = read_back(lg, dg), read_back(lw, dw)
    for name, _ in LAYOUT + DERIVED:
        if (name in ("blk", "blk_ub") and lw.n_blocks == 0) or (name == "champ" and dw.n_champ == 0):
            continue
        assert ag[name].tobytes() == aw[name].tobytes(), f"{what}: {name} differs"


def _same_index(got, want, what):
    _same_arrays(got.layout(), got.derived(), want.layout(), want.derived(), what)
    a, w = got.info(), want.info()
    for f, _ in type(w)._fields_:
        assert getattr(a, f) == getattr(w, f), f"{what}: info.{f}"
    assert np.array_equal(got.df(), want.df()), f"{what}: df"


def _keyed(rng, elem_off, elem_term, keys_of_term):
    """The documents with term t written as keys_of_term[t], each document's elements re-sorted by key."""
    off = np.asarray(elem_off, np.int64)
    doc = np.repeat(np.arange(len(off) - 1), np.diff(off))
    key = keys_of_term[np.asarray(elem_term, np.int64)]
    hi, lo = key_words(key)
    order = np.lexsort((lo, hi, doc))
    return key[order], order


def _random_keys(rng, n):
    k = rng.integers(0, 256, size=(n, 16), dtype=np.uint8)
    k[:, 0] |= 0x80 * (np.arange(n) % 2).astype(np.uint8)            # half of them with a first byte >= 0x80
    assert len(np.unique(k, axis=0)) == n
    return k


def _build_both(m, docs, k1=1.2, b=0.75, payload=None):
    """(from documents, from the Segment's CSR, the Segment)."""
    s = segment(**{f: docs[f] for f in docs if f != "n_terms"}, n_terms=docs.get("n_terms", 0))
    got = m.Index.from_documents(**docs, payload=payload, k1=k1, b=b)
    want = m.Index(**csr_kwargs(s), k1=k1, b=b, payload=payload)
    return got, want, s


def _small_cases(rng):
    """(name, documents, k1, b, payload) of the hand-made shapes, keyless and keyed."""
    cases = []
    # empty documents among others; a term in every document; unused ordinals, n_terms - 1 among them
    n, T = 300, 50
    lens = rng.integers(0, 9, n)
    lens[[0, 7, 299]] = 0
    terms = [np.union1d([3], rng.choice(T - 2, size=l, replace=False)) if l else np.zeros(0, np.int64) for l in lens]
    terms[0], terms[7], terms[299] = np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64)
    off = np.concatenate([[0], np.cumsum([len(t) for t in terms])]).astype(np.uint64)
    term = np.concatenate(terms).astype(np.uint32)
    unused = np.setdiff1d(np.arange(T), term)
    assert T - 1 in unused and T - 2 in unused
    tf = rng.integers(1, 40, len(term)).astype(np.uint32)
    tf[:5] = (1 << 24) - 1
    cases.append(("mixed", dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=T), 1.2, 0.75, None))
    pay = rng.integers(0, 1 << 16, n * 3).astype(np.uint16)
    cases.append(("mixed payload k1 b", dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=T), 2.0, 0.3, pay))
    cases.append(("mixed b=0", dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=T), 0.0, 0.0, pay))
    keys = _random_keys(rng, T)
    kk, order = _keyed(rng, off, term, keys)
    cases.append(("mixed keyed", dict(elem_off=off, elem_tf=tf[order], elem_key=kk), 1.5, 1.0, pay))
    # all documents empty but one
    off1 = np.zeros(101, np.uint64)
    off1[51:] = 4
    t1 = np.array([0, 5, 6, 9], np.uint32)
    cases.append(("one document", dict(elem_off=off1, elem_tf=np.array([1, 2, 3, 4], np.uint32), elem_term=t1,
                                       n_terms=12), 1.2, 0.75, None))
    k4 = keys[:4][np.lexsort(key_words(keys[:4])[::-1])]            # ascending bytewise: a Document
    cases.append(("one document keyed", dict(elem_off=off1, elem_tf=np.array([1, 2, 3, 4], np.uint32), elem_key=k4),
                  1.2, 0.75, None))
    # T = 1: one term in every other document
    offt = np.concatenate([[0], np.cumsum(np.arange(500) % 2)]).astype(np.uint64)
    cases.append(("T=1", dict(elem_off=offt, elem_tf=rng.integers(1, 9, 250).astype(np.uint32),
                              elem_term=np.zeros(250, np.uint32), n_terms=1), 1.2, 0.75, None))
    cases.append(("T=1 keyed", dict(elem_off=offt, elem_tf=rng.integers(1, 9, 250).astype(np.uint32),
                                    elem_key=np.repeat(keys[:1], 250, axis=0)), 1.2, 0.75, None))
    # keys that differ only in their first byte or only in their last byte, bytes >= 0x80
    base = np.full(16, 0x41, np.uint8)
    ks = []
    for v in (0x00, 0x01, 0x7F, 0x80, 0xFF):
        a = base.copy()
        a[0] = v
        ks.append(a)
        a = base.copy()
        a[15] = v
        ks.append(a)
    ks = np.unique(np.array(ks), axis=0)
    rng.shuffle(ks)
    nd = 400
    lens = rng.integers(0, len(ks) + 1, nd)
    per = [np.sort(rng.choice(len(ks), size=l, replace=False)) for l in lens]
    offk = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    tk = np.concatenate(per).astype(np.uint32)
    kk, order = _keyed(rng, offk, tk, ks)
    tfk = rng.integers(1, 300, len(tk)).astype(np.uint32)
    cases.append(("edge keys", dict(elem_off=offk, elem_tf=tfk[order], elem_key=kk), 1.2, 0.75, None))
    return cases


@pytest.mark.parametrize("i", range(9))
def test_small_documents_equal_the_segment_build(m, i):
    name, docs, k1, b, pay = _small_cases(np.random.default_rng(7))[i]
    got, want, s = _build_both(m, docs, k1, b, pay)
    _same_index(got, want, name)
    if s.term_keys is not None:
        assert np.array_equal(got.lookup_terms(s.term_keys), np.arange(s.n_terms, dtype=np.uint32)), name
        a, ax = got.export_blocks(term_keys=True)
        w, wx = want.export_blocks(term_keys=True)
        a.update(ax)
        w.update(wx)
        for key in w:
            x, y = a[key], w[key]
            assert (x is None and y is None) or (np.asarray(x).tobytes() == np.asarray(y).tobytes()), f"{name}: {key}"


def _synth_docs(m, seed, n, vocab, lmin, lmax, zipf):
    c = m.synth_corpus(seed, n, vocab, lmin, lmax, zipf)
    off, term, tf = documents_of_csr(c.n_docs, c.post_off, c.post_doc, c.post_tf)
    return c, dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=c.n_terms)


@pytest.mark.parametrize("keyed", [False, True])
def test_synthetic_corpus_rows_and_oracle(m, orc, keyed):
    c, docs = _synth_docs(m, 22, 30000, 5000, 16, 96, 1.0)
    if keyed:
        rng = np.random.default_rng(3)
        kk, order = _keyed(rng, docs["elem_off"], docs["elem_term"], _random_keys(rng, c.n_terms))
        docs = dict(elem_off=docs["elem_off"], elem_tf=docs["elem_tf"][order], elem_key=kk)
    got, want, s = _build_both(m, docs)
    if not keyed:
        for f in ("doc_len", "post_off", "post_doc", "post_tf"):
            assert np.array_equal(getattr(s, f), getattr(c, f)), f"the Segment restates the synthetic CSR: {f}"
    _same_index(got, want, f"synthetic keyed={keyed}")
    q_off, q_terms = m.synth_queries(5, 80, s.n_terms, 1, 8, s.post_off)
    oix = oracle_index(orc, s)
    for k in (1, 10, 100, 1000):
        a = got.search_batch(q_off, q_terms, k, want_payload=True)
        same_rows(a, want.search_batch(q_off, q_terms, k, want_payload=True), f"k={k}")
        compare(a, oix, q_off, q_terms, k, what=f"oracle k={k}")


def test_chunks_documents_straddle_and_terms_span(m):
    """More than three chunks: documents cut by chunk boundaries, and a term (in every document) whose postings come from
    every chunk."""
    rng = np.random.default_rng(11)
    n, vocab = 150_000, 20_000
    lens = rng.integers(60, 200, n)
    E = int(lens.sum())
    assert E > 3 * CHUNK + CHUNK // 2
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    term = np.empty(E, np.uint32)
    for d0 in range(0, n, 10_000):                                  # term 0 in every document, the rest distinct
        for d in range(d0, min(n, d0 + 10_000)):
            t = rng.choice(vocab - 1, size=lens[d] - 1, replace=False) + 1
            t.sort()
            term[off[d]] = 0
            term[off[d] + 1:off[d + 1]] = t
    tf = rng.integers(1, 50, E).astype(np.uint32)
    for c in range(1, 4):
        d = int(np.searchsorted(off, c * CHUNK, side="right")) - 1
        assert off[d] < c * CHUNK < off[d + 1], f"document {d} straddles chunk boundary {c}"
    docs = dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=vocab)
    got, want, s = _build_both(m, docs)
    assert s.post_off[1] == n                                       # term 0: one posting per document, every chunk
    _same_index(got, want, "four-plus chunks")
    q_off, q_terms = query_csr([[0], [0, 5], [7, 11, 13], list(range(1, 9))])
    for k in (1, 10, 100, 1000):
        same_rows(got.search_batch(q_off, q_terms, k), want.search_batch(q_off, q_terms, k), f"k={k}")


def test_golden_passages_keyed(m, golden):
    intern = __import__(m.__name__ + ".bm25x", fromlist=["x"]).intern
    seed = bytes(range(32))
    for ids, rank in ((list(range(1, 11)), "ranking_full_index"), ([2, 4, 6, 8, 10], "ranking_even_ids"),
                      ([1, 3, 5, 7, 9], "ranking_odd_ids")):
        keys, tfs, off = [], [], [0]
        for i in ids:
            counts = {}
            for w in golden["doc_lexemes"][i - 1]:
                kw = intern(seed, w.encode())
                counts[kw] = counts.get(kw, 0) + 1
            for kw in sorted(counts):                                # bytewise ascending: a Document
                keys.append(np.frombuffer(kw, np.uint8))
                tfs.append(counts[kw])
            off.append(len(keys))
        ix = m.Index.from_documents(np.array(off, np.uint64), np.array(tfs, np.uint32), elem_key=np.array(keys))
        assert ix.info().sum_doc_len == sum(golden["doc_lengths"][i - 1] for i in ids)
        t = ix.lookup_terms(np.frombuffer(intern(seed, b"postgresql"), np.uint8))
        docs, _ = ix.search(t, 10)
        assert [ids[d] for d in docs] == golden[rank], rank
        ix.close()


@pytest.mark.parametrize("keyed", [False, True])
@pytest.mark.parametrize("S, bounds", [(2, None), (4, None), (2, "given"), (4, "given")])
def test_sharded_equals_sharded_create(m, orc, keyed, S, bounds):
    c, docs = _synth_docs(m, 23, 5000, 40, 5, 400, 1.1)
    if keyed:
        rng = np.random.default_rng(5)
        kk, order = _keyed(rng, docs["elem_off"], docs["elem_term"], _random_keys(rng, c.n_terms))
        docs = dict(elem_off=docs["elem_off"], elem_tf=docs["elem_tf"][order], elem_key=kk)
    s = segment(**{f: docs[f] for f in docs if f != "n_terms"}, n_terms=docs.get("n_terms", 0))
    b = None if bounds is None else np.linspace(0, s.n_docs, S + 1).astype(np.uint32)
    got = m.ShardedIndex.from_documents(**docs, n_shards=S, doc_bounds=b, k1=1.4, b=0.6)
    want = m.ShardedIndex(**csr_kwargs(s), n_shards=S, doc_bounds=b, k1=1.4, b=0.6)
    ix = m.Index(**csr_kwargs(s), k1=1.4, b=0.6)
    what = f"S={S} bounds={bounds} keyed={keyed}"
    assert np.array_equal(got.doc_bounds(), want.doc_bounds()), what
    for sh in range(S):
        (lg, dg), (lw, dw) = got.shard_arrays(sh), want.shard_arrays(sh)
        _same_arrays(lg, dg, lw, dw, f"{what} shard {sh}")
    a, w = got.info(), want.info()
    for f, _ in type(w)._fields_:
        assert getattr(a, f) == getattr(w, f), f"{what}: info.{f}"
    check_shards(m, orc, dict(n_docs=s.n_docs, doc_len=s.doc_len, n_terms=s.n_terms, post_off=s.post_off,
                              post_doc=s.post_doc, post_tf=s.post_tf), got, ix, 1.4, 0.6, what)
    if keyed:
        assert np.array_equal(got.lookup_terms(s.term_keys), np.arange(s.n_terms, dtype=np.uint32)), what
    q_off, q_terms = m.synth_queries(9, 60, s.n_terms, 1, 8, s.post_off)
    for k in (1, 10, 100, 1000):
        same_rows(got.search_batch(q_off, q_terms, k, want_payload=True),
                  ix.search_batch(q_off, q_terms, k, want_payload=True), f"{what} k={k}")


def test_device_refusals_leave_no_memory(m):
    c, docs = _synth_docs(m, 0xB25C0DE1, 1000, 1000, 32, 32, 0.0)
    Index, Sharded = m.Index, m.ShardedIndex
    before = free_bytes()
    code, msg = refused(m, lambda: Index.from_documents(**docs, device=99))
    assert code == 2 and "bm25x_index_create_from_documents: CUDA device 99 not available" in msg
    code, msg = refused(m, lambda: Sharded.from_documents(**docs, n_shards=2, devices=[0, 99]))
    assert code == 2 and "bm25x_index_create_sharded_from_documents: CUDA device 99 not available" in msg
    bad = docs["elem_tf"].copy()
    bad[-1] = 0
    code, _ = refused(m, lambda: Index.from_documents(**dict(docs, elem_tf=bad)))
    assert code == 1
    assert free_bytes() == before
