"""The builds from documents and tsvectors at the sizes where their chunkers cut: the keyed vocabulary pass compacting
every chunk, documents cut by every chunk boundary, a sharded build whose shards start mid-chunk or hold no element, a
document whose Σ tf passes 2^32 - 1, and tsvector casts cut by lexeme bytes, by a vector larger than a chunk and by a
saturating merge longer than 2^32 / 65535 entries.

Every fixture has a CPU test (no device) that asserts on the restated chunk schedules (util_documents.vocab_schedule,
util_tsvector.cast_cuts) that it reaches the branch it is there for.  The GPU tests compare with restatements that share
no code with the device path: the Segment of the documents (util_documents.segment) built by the CSR build, the oracle's
rows, and the host cast over bm25x_intern (util_tsvector.cast)."""
import numpy as np
import pytest

from util_documents import CHUNK, csr_kwargs, key_words, segment, vocab_schedule
from util_index import DERIVED, LAYOUT, SCALARS, fieldnorms, read_back
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import compare, oracle_index, query_csr, same_rows
from util_tsvector import CHUNK_BYTES, CHUNK_ENT, assemble, byte_cut_batch, cast, cast_cuts

SEED = bytes((11 * i + 5) & 0xFF for i in range(32))
P0, P1 = 49999, 50021          # primes: the id ranges of the documents before and inside the last chunk
EMPTY = (45_000, 45_500)       # the empty documents of the corpus (shard 1 of the sharded build)
EDGE = (0x00, 0x7F, 0x80, 0xFF)


def _bm(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


# ---- the keyed corpus of 3-4 chunks over a small vocabulary ----

def _corpus():
    """About 3.7 chunks of documents of 60..200 distinct terms: term 0 in every non-empty one, terms P0 + 1 .. P1 only in
    the documents that start in the last chunk, documents EMPTY empty.  Terms 1..8 are keys that differ from one another
    only in byte 0 or only in byte 15.  Returns dict(off, doc, term, tf, keys) with each document's elements in term
    order; keyed() and keyless() order them as each build takes them."""
    rng = np.random.default_rng(41)
    n = 120_000
    lens = rng.integers(60, 201, n)
    lens[EMPTY[0]:EMPTY[1]] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    E = int(off[-1])
    doc = np.repeat(np.arange(n, dtype=np.int64), lens)
    j = np.arange(E, dtype=np.int64) - off[:-1].astype(np.int64)[doc]
    P = np.where(off[:-1] >= 3 * CHUNK, P1, P0)
    start, stride = rng.integers(0, P), rng.integers(1, P)
    # element 0 of a document is term 0; element j > 0 is 1 + (start + j * stride) mod P: distinct for j < P
    term = np.where(j == 0, 0, 1 + (start[doc] + j * stride[doc]) % P[doc]).astype(np.uint32)
    T = P1 + 1
    keys = rng.integers(0, 256, (T, 16), dtype=np.uint8)
    base = np.full(16, 0x41, np.uint8)
    for i, v in enumerate(EDGE):
        keys[1 + 2 * i], keys[2 + 2 * i] = base, base
        keys[1 + 2 * i, 0], keys[2 + 2 * i, 15] = v, v
    assert len(np.unique(keys, axis=0)) == T
    tf = rng.integers(1, 50, E).astype(np.uint32)
    order = np.argsort((doc.astype(np.uint64) << np.uint64(32)) | term.astype(np.uint64), kind="stable")
    return dict(off=off, doc=doc[order], term=term[order], tf=tf[order], keys=keys)


def _rank(c):
    """Each term's rank among the keys, ascending bytewise."""
    hi, lo = key_words(c["keys"])
    rank = np.empty(len(hi), np.uint64)
    rank[np.lexsort((lo, hi))] = np.arange(len(hi), dtype=np.uint64)
    return rank


def _keyed(c):
    """The corpus as keyed documents: each document's keys ascending bytewise."""
    order = np.argsort((c["doc"].astype(np.uint64) << np.uint64(32)) | _rank(c)[c["term"]], kind="stable")
    return dict(elem_off=c["off"], elem_tf=c["tf"][order], elem_key=c["keys"][c["term"][order]])


def _keyless(c):
    return dict(elem_off=c["off"], elem_tf=c["tf"], elem_term=c["term"], n_terms=len(c["keys"]))


def _bounds(c):
    return np.array([0, EMPTY[0], EMPTY[1], len(c["off"]) - 1], np.uint32)


@pytest.fixture(scope="module")
def corpus():
    return _corpus()


def test_corpus_compacts_every_chunk_and_cuts_documents(corpus):
    c = corpus
    off = c["off"].astype(np.int64)
    E = int(off[-1])
    assert 3 * CHUNK < E < 4 * CHUNK
    ev = vocab_schedule(_keyed(c)["elem_key"])
    # vocab_pass: the list grows once (chunk 0, nothing kept) and, the vocabulary being smaller than a chunk, every chunk
    # compacts its own appended entries (A = CHUNK, then the partial last chunk): no chunk is deferred
    assert ev[0] == ("grow", 0, 2 * CHUNK, 0)
    assert [e for e in ev if e[0] != "grow"] == [("compact", i, min(CHUNK, E - i * CHUNK)) for i in range(4)]
    # every chunk boundary cuts a document
    for b in range(1, 4):
        d = int(np.searchsorted(off, b * CHUNK, side="right")) - 1
        assert off[d] < b * CHUNK < off[d + 1], f"document {d} straddles chunk boundary {b}"
    # term 0 in every non-empty document; terms P0 + 1 .. P1 first seen in the last chunk, all of them
    first = np.full(len(c["keys"]), E, np.int64)
    np.minimum.at(first, c["term"].astype(np.int64), np.arange(E))
    assert (first[P0 + 1:] >= 3 * CHUNK).all() and (first[P0 + 1:] < E).all() and (first[:P0 + 1] < 3 * CHUNK).all()
    assert np.count_nonzero(c["term"] == 0) == np.count_nonzero(np.diff(off))
    assert (first[1:9] < E).all()                                   # the byte-0 / byte-15 keys are used


def test_sharded_bounds_cut_chunks_and_hold_an_empty_shard(corpus):
    off = corpus["off"].astype(np.int64)
    b = _bounds(corpus)
    e = off[b]
    assert CHUNK < e[1] < 2 * CHUNK and e[1] % CHUNK                # shard 0 ends inside chunk 1
    assert b[2] > b[1] and e[2] == e[1]                             # shard 1: documents, no element (invert's ch == 0)
    assert e[3] - e[2] > 2 * CHUNK and e[2] % CHUNK                 # shard 2: starts mid-chunk, spans over 2 chunks
    assert (e[3] - e[2]) % CHUNK                                    # and ends in a partial chunk of its own


def _same_arrays(lg, dg, lw, dw, what):
    for name in SCALARS:
        assert getattr(lg, name) == getattr(lw, name), f"{what}: {name} {getattr(lg, name)} != {getattr(lw, name)}"
    assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min, what
    ag, aw = read_back(lg, dg), read_back(lw, dw)
    for name, _ in LAYOUT + DERIVED:
        if (name in ("blk", "blk_ub") and lw.n_blocks == 0) or (name == "champ" and dw.n_champ == 0):
            continue
        assert ag[name].tobytes() == aw[name].tobytes(), f"{what}: {name} differs"


def _same_info(got, want, what):
    a, w = got.info(), want.info()
    for f, _ in type(w)._fields_:
        assert getattr(a, f) == getattr(w, f), f"{what}: info.{f}"


def _same_index(got, want, what):
    _same_arrays(got.layout(), got.derived(), want.layout(), want.derived(), what)
    _same_info(got, want, what)
    assert np.array_equal(got.df(), want.df()), f"{what}: df"


def _queries(rng, s, must, nq=300):
    """nq queries of 1..8 live terms, every one of them holding one of `must` (the shared key, the late keys, the edge
    keys)."""
    df = np.diff(s.post_off.astype(np.int64))
    live = np.flatnonzero(df > 0)
    qs = []
    for i in range(nq):
        q = set(rng.choice(live, size=int(rng.integers(0, 8)), replace=False).tolist())
        q.add(int(must[i % len(must)]))
        qs.append(sorted(q))
    return query_csr(qs)


def _rows_and_oracle(orc, got, want, s, must, what, rng_seed=3):
    q_off, q_terms = _queries(np.random.default_rng(rng_seed), s, must)
    oix = oracle_index(orc, s)
    for k in (1, 10, 100, 1000):
        a = got.search_batch(q_off, q_terms, k, want_payload=True)
        same_rows(a, want.search_batch(q_off, q_terms, k, want_payload=True), f"{what} k={k}")
        compare(a, oix, q_off, q_terms, k, what=f"{what} oracle k={k}")


def _must(c, keyed):
    """The terms every query holds one of, as the Segment numbers them: the shared term, the edge keys, the late terms."""
    t = np.concatenate([[0], np.arange(1, 9), np.arange(P0 + 1, P1 + 1)])
    return _rank(c)[t] if keyed else t


def _segment(c, docs):
    s = segment(**{f: docs[f] for f in docs if f != "n_terms"}, n_terms=docs.get("n_terms", 0))
    assert s.n_terms == len(c["keys"])                               # every term used: ordinal = rank of its key
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("keyed", [True, False])
def test_documents_of_four_chunks_equal_the_segment_build(m, orc, corpus, keyed):
    docs = _keyed(corpus) if keyed else _keyless(corpus)
    s = _segment(corpus, docs)
    got = m.Index.from_documents(**docs)                            # the oracle's k1 and b
    want = m.Index(**csr_kwargs(s))
    what = f"keyed={keyed}"
    t0 = int(_must(corpus, keyed)[0])                               # the shared term: postings from every chunk
    assert s.post_off[t0 + 1] - s.post_off[t0] == np.count_nonzero(np.diff(corpus["off"].astype(np.int64)))
    _same_index(got, want, what)
    if keyed:
        assert np.array_equal(got.lookup_terms(s.term_keys), np.arange(s.n_terms, dtype=np.uint32)), what
    _rows_and_oracle(orc, got, want, s, _must(corpus, keyed), what)


@pytest.mark.gpu
@pytest.mark.parametrize("keyed", [True, False])
def test_sharded_documents_equal_sharded_create(m, orc, corpus, keyed):
    docs = _keyed(corpus) if keyed else _keyless(corpus)
    s = _segment(corpus, docs)
    b = _bounds(corpus)
    got = m.ShardedIndex.from_documents(**docs, n_shards=3, doc_bounds=b, k1=1.1, b=0.8)
    want = m.ShardedIndex(**csr_kwargs(s), n_shards=3, doc_bounds=b, k1=1.1, b=0.8)
    ix = m.Index(**csr_kwargs(s), k1=1.1, b=0.8)
    what = f"sharded keyed={keyed}"
    assert np.array_equal(got.doc_bounds(), b) and np.array_equal(want.doc_bounds(), b), what
    for sh in range(3):
        (lg, dg), (lw, dw) = got.shard_arrays(sh), want.shard_arrays(sh)
        _same_arrays(lg, dg, lw, dw, f"{what} shard {sh}")
    assert got.shard_arrays(1)[0].n_postings == 0, what
    _same_info(got, want, what)
    if keyed:
        assert np.array_equal(got.lookup_terms(s.term_keys), np.arange(s.n_terms, dtype=np.uint32)), what
    q_off, q_terms = _queries(np.random.default_rng(5), s, _must(corpus, keyed))
    for k in (1, 10, 100, 1000):
        same_rows(got.search_batch(q_off, q_terms, k, want_payload=True),
                  ix.search_batch(q_off, q_terms, k, want_payload=True), f"{what} k={k}")


# ---- a document whose Σ tf passes 2^32 - 1 ----

BIG_DOC, BIG_ELEMS, BIG_TF = 17, 300, (1 << 24) - 1


def _saturating_documents():
    """60 documents of 1..20 terms over 500 terms; document BIG_DOC holds BIG_ELEMS terms of tf 2^24 - 1."""
    rng = np.random.default_rng(13)
    terms = [np.sort(rng.choice(500, size=int(rng.integers(1, 21)), replace=False)) for _ in range(60)]
    terms[BIG_DOC] = np.sort(rng.choice(500, size=BIG_ELEMS, replace=False))
    tfs = [rng.integers(1, 30, len(t)) for t in terms]
    tfs[BIG_DOC] = np.full(BIG_ELEMS, BIG_TF)
    off = np.concatenate([[0], np.cumsum([len(t) for t in terms])]).astype(np.uint64)
    return off, np.concatenate(terms).astype(np.uint32), np.concatenate(tfs).astype(np.uint32), 500


# 257 lexemes in one vector, each in 256 entries of 65535 positions: merged tf 256 * 65535 < 2^24, their sum > 2^32
SAT_LEX, SAT_REP, SAT_CNT = 257, 256, 65535


def _saturating_tsvectors():
    """Small vectors beside vector 3, which holds SAT_LEX two-byte lexemes back to back with their u16 counts (the cast
    reads the count after each lexeme, never the positions)."""
    rng = np.random.default_rng(14)
    vectors = []
    for v in range(8):
        if v == 3:
            lex = [bytes([97 + i // 26, 97 + i % 26]) for i in range(SAT_LEX)]
            area = b"".join(x + SAT_CNT.to_bytes(2, "little") for x in lex)
            ents = [((4 * i) << 12) | (2 << 1) | 1 for i in range(SAT_LEX)] * SAT_REP
        else:
            k = int(rng.integers(1, 12))
            area, ents = b"", []
            for i in range(k):
                x = b"w%d" % int(rng.integers(0, 40))
                at = len(area)
                area += x + (b"\0" if len(x) % 2 else b"") + int(rng.integers(1, 9)).to_bytes(2, "little")
                ents.append((at << 12) | (len(x) << 1) | 1)
        vectors.append((np.frombuffer(area, np.uint8), np.array(ents, np.uint32)))
    return assemble(vectors)


def test_saturating_fixtures_pass_two_to_the_32(orc):
    off, term, tf, _ = _saturating_documents()
    s = segment(off, tf, elem_term=term, n_terms=500)
    assert int(tf[off[BIG_DOC]:off[BIG_DOC + 1]].astype(np.uint64).sum()) > 0xFFFFFFFF
    assert s.doc_len[BIG_DOC] == 0xFFFFFFFF and (s.doc_len[np.arange(60) != BIG_DOC] < 1000).all()
    tsv = _saturating_tsvectors()
    c_off, _, c_tf = cast(None, SEED, tsv, keys=_copy_keys(tsv))
    row = c_tf[c_off[3]:c_off[4]]
    assert len(row) == SAT_LEX and (row == SAT_REP * SAT_CNT).all() and SAT_REP * SAT_CNT < (1 << 24)
    assert int(row.astype(np.uint64).sum()) > 0xFFFFFFFF
    # truncated to u32, the length would be 16 711 424: a different fieldnorm
    fn = fieldnorms(orc, np.array([0xFFFFFFFF, int(row.astype(np.uint64).sum()) & 0xFFFFFFFF]))
    assert fn[0] != fn[1]


def _copy_keys(tsv):
    """Keys of entries whose lexemes are shorter than 16 bytes and NUL-free: the lexeme zero-padded (vector::intern's
    copy path), computed in slices of entries."""
    ent_off = np.asarray(tsv["ent_off"], np.int64)
    e = np.asarray(tsv["entries"], np.uint32).astype(np.int64)
    vec = np.repeat(np.arange(len(ent_off) - 1), np.diff(ent_off))
    start = np.asarray(tsv["byte_off"], np.int64)[:-1][vec] + (e >> 12)
    length = (e >> 1) & 0x7FF
    data = np.asarray(tsv["data"], np.uint8)
    keys = np.zeros((len(e), 16), np.uint8)
    j = np.arange(15)
    for a in range(0, len(e), 1 << 20):
        st, ln = start[a:a + (1 << 20)], length[a:a + (1 << 20)]
        assert (ln < 16).all()
        mask = j[None, :] < ln[:, None]
        got = np.where(mask, data[np.where(mask, st[:, None] + j[None, :], 0)], 0).astype(np.uint8)
        assert (got[mask] != 0).all()
        keys[a:a + len(ln), :15] = got
    return keys


def _check_saturated_index(orc, got, want, s, big, what):
    _same_index(got, want, what)
    assert s.doc_len[big] == 0xFFFFFFFF, what
    fn = read_back(got.layout(), got.derived())["fieldnorm"]
    assert fn[big] == fieldnorms(orc, np.array([0xFFFFFFFF]))[0], what
    assert got.info().sum_doc_len == int(s.doc_len.astype(np.uint64).sum()), what
    rng = np.random.default_rng(8)
    df = np.diff(s.post_off.astype(np.int64))
    live = np.flatnonzero(df > 0)
    qs = [sorted(set(rng.choice(live, size=int(rng.integers(1, 6)), replace=False).tolist())) for _ in range(80)]
    q_off, q_terms = query_csr(qs)
    oix = oracle_index(orc, s)
    for k in (1, 10, 100, 1000):
        compare(got.search_batch(q_off, q_terms, k), oix, q_off, q_terms, k, what=f"{what} k={k}")


@pytest.mark.gpu
@pytest.mark.parametrize("keyed", [False, True])
def test_document_length_saturates_from_documents(m, orc, keyed):
    off, term, tf, T = _saturating_documents()
    if keyed:
        keys = np.random.default_rng(2).integers(0, 256, (T, 16), dtype=np.uint8)
        hi, lo = key_words(keys)
        rank = np.empty(T, np.int64)
        rank[np.lexsort((lo, hi))] = np.arange(T)
        doc = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
        order = np.lexsort((rank[term], doc))
        docs = dict(elem_off=off, elem_tf=tf[order], elem_key=keys[term[order]])
    else:
        docs = dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=T)
    s = segment(**{f: docs[f] for f in docs if f != "n_terms"}, n_terms=docs.get("n_terms", 0))
    got = m.Index.from_documents(**docs)
    want = m.Index(**csr_kwargs(s))
    _check_saturated_index(orc, got, want, s, BIG_DOC, f"documents keyed={keyed}")


@pytest.mark.gpu
def test_document_length_saturates_from_tsvectors(m, orc):
    tsv = _saturating_tsvectors()
    c_off, c_keys, c_tf = cast(_bm(m).intern, SEED, tsv)
    s = segment(c_off, c_tf, elem_key=c_keys)
    got = m.Index.from_tsvectors(SEED, **tsv)
    want = m.Index(**csr_kwargs(s))
    _check_saturated_index(orc, got, want, s, 3, "tsvectors")


# ---- tsvector casts at every chunk cut ----

def _same_cast(m, tsv, what, keys=None):
    bm = _bm(m)
    for as_query in (False, True):
        got = bm.cast_tsvectors(SEED, **tsv, as_query=as_query)
        want = cast(bm.intern, SEED, tsv, as_query=as_query, keys=keys)
        w = f"{what} query={as_query}"
        assert np.array_equal(got[0], want[0]), f"{w}: offsets"
        assert got[1].tobytes() == want[1].tobytes(), f"{w}: keys"
        assert (got[2] is None) == as_query and (as_query or np.array_equal(got[2], want[2])), f"{w}: tf"


def _same_build_and_queries(m, tsv, what, keys=None):
    """from_tsvectors against the CSR build of the Segment of the restated cast; tsvector_queries of the same batch
    against lookup_terms of the restated query keys; search rows alike."""
    bm = _bm(m)
    off, k, tf = cast(bm.intern, SEED, tsv, keys=keys)
    s = segment(off, tf, elem_key=k)
    got = m.Index.from_tsvectors(SEED, **tsv)
    want = m.Index(**csr_kwargs(s))
    _same_index(got, want, what)
    q_off, q_terms = got.tsvector_queries(SEED, **tsv)
    qo, qk, _ = cast(bm.intern, SEED, tsv, as_query=True, keys=keys)
    assert np.array_equal(q_off, qo.astype(np.uint32)), f"{what}: query offsets"
    assert np.array_equal(q_terms, want.lookup_terms(qk) if len(qk) else np.zeros(0, np.uint32)), f"{what}: query terms"
    pick = np.flatnonzero(np.diff(q_off.astype(np.int64)) > 0)[::max(1, len(q_off) // 200)][:200]
    qs = [q_terms[q_off[i]:q_off[i + 1]][:8] for i in pick]
    a_off, a_terms = query_csr(qs)
    for kk in (1, 10, 100, 1000):
        same_rows(got.search_batch(a_off, a_terms, kk, want_payload=True),
                  want.search_batch(a_off, a_terms, kk, want_payload=True), f"{what} k={kk}")
    return got


def _window_batch():
    """One vector of CHUNK_ENT + 3 entries and one of exactly CHUNK_ENT, small vectors around them and an empty one after
    the exact one.  Each vector's entries are windows of 3..15 bytes of its own area of random bytes 1..255 (the copy
    path; every u16 count after a window is non-zero), the big ones' areas just under 1 MiB."""
    rng = np.random.default_rng(22)
    lens = [9, 30, 1, CHUNK_ENT + 3, 12, 40, CHUNK_ENT, 0, 7, 25]
    vectors = []
    for n in lens:
        size = (1 << 20) - 64 if n > 1000 else 4096
        area = rng.integers(1, 256, size, dtype=np.uint8)
        ln = rng.integers(3, 16, n)
        pos = rng.integers(0, size - 18, n)
        vectors.append((area, ((pos << 12) | (ln << 1) | 1).astype(np.uint32)))
    return assemble(vectors)


def _saturating_merge_batch(reps, before):
    """Vector 1 holds one lexeme in `reps` entries of 65535 positions (a merged sum past 2^32 - 1) and a few others;
    vector 0 holds `before` entries, so the run starts at another offset inside a sort tile."""
    rng = np.random.default_rng(reps)
    lex = [b"w%d" % i for i in range(50)]

    def vector(entries):
        area, ents = bytearray(), []
        for x, cnt in entries:
            at = len(area)
            area += x + (b"\0" if len(x) % 2 else b"") + cnt.to_bytes(2, "little")
            ents.append((at << 12) | (len(x) << 1) | 1)
        return np.frombuffer(bytes(area), np.uint8), np.array(ents, np.uint32)

    v0 = vector([(lex[int(i)], int(rng.integers(1, 100))) for i in rng.integers(0, 50, before)])
    area, ents = vector([(b"saturate", 65535), (b"a", 3), (b"zz", 2)])
    ents = np.concatenate([ents[1:2], np.repeat(ents[:1], reps), ents[2:]])
    rng.shuffle(ents)
    v2 = vector([(lex[3], 1), (b"saturate", 5)])
    return assemble([v0, (area, ents), v2])


def test_byte_cut_batch_cuts_on_bytes():
    tsv, _, _ = byte_cut_batch()
    cuts = cast_cuts(tsv)
    byt = tsv["byte_off"].astype(np.int64)
    assert [(a, b, r) for a, b, r, _ in cuts] == [(0, 64, "bytes"), (64, 127, "bytes"), (127, 133, "end")]
    assert byt[64] - byt[0] == CHUNK_BYTES                          # an area that ends exactly at the limit: taken
    assert byt[128] - byt[64] == CHUNK_BYTES + 1                    # one byte past it: cut before
    assert all(ne < CHUNK_ENT // 100 for *_, ne in cuts)


def test_window_batch_has_a_vector_larger_than_a_chunk():
    tsv = _window_batch()
    cuts = cast_cuts(tsv)
    assert [(a, b, r) for a, b, r, _ in cuts] == [(0, 3, "entries"), (3, 4, "single"), (4, 6, "entries"),
                                                 (6, 8, "entries"), (8, 10, "end")]
    assert cuts[1][3] == CHUNK_ENT + 3 and cuts[3][3] == CHUNK_ENT
    assert tsv["data"].nbytes < 4 << 20 and (tsv["byte_off"][4] - tsv["byte_off"][3]) <= 1 << 20
    off, _, tf = cast(None, SEED, tsv, keys=_copy_keys(tsv))
    assert tf.max() < (1 << 24) and tf.min() > 0                    # the build takes it


@pytest.mark.parametrize("reps, before", [(65_538, 1000), (70_001, 3333)])
def test_saturating_merge_batch_passes_two_to_the_32(reps, before):
    tsv = _saturating_merge_batch(reps, before)
    assert reps * 65535 > 0xFFFFFFFF
    assert [r for *_, r, _ in cast_cuts(tsv)] == ["end"]
    off, keys, tf = cast(None, SEED, tsv, keys=_copy_keys(tsv))
    row = slice(int(off[1]), int(off[2]))
    assert keys[row].tobytes().count(b"saturate") == 1 and tf[row].max() == 0xFFFFFFFF


@pytest.mark.gpu
def test_cast_build_and_queries_cut_by_bytes(m):
    tsv, words, wid = byte_cut_batch()
    bm = _bm(m)
    wkeys = np.array([np.frombuffer(bm.intern(SEED, w), np.uint8) for w in words])
    keys = wkeys[wid]
    _same_cast(m, tsv, "bytes", keys=keys)
    _same_build_and_queries(m, tsv, "bytes", keys=keys)


@pytest.mark.gpu
def test_cast_build_and_queries_of_a_vector_larger_than_a_chunk(m):
    tsv = _window_batch()
    keys = _copy_keys(tsv)
    _same_cast(m, tsv, "windows", keys=keys)
    _same_build_and_queries(m, tsv, "windows", keys=keys)


@pytest.mark.gpu
@pytest.mark.parametrize("reps, before", [(65_538, 1000), (70_001, 3333)])
def test_cast_saturating_merge(m, reps, before):
    tsv = _saturating_merge_batch(reps, before)
    _same_cast(m, tsv, f"saturate {reps}", keys=_copy_keys(tsv))
    off, keys, tf = _bm(m).cast_tsvectors(SEED, **tsv)
    row = slice(int(off[1]), int(off[2]))
    assert tf[row].max() == 0xFFFFFFFF
