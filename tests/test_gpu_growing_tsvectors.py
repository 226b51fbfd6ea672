"""GPU: tsvector inserts into the growing segment (bm25x_growing_insert_tsvectors) against a twin: a second segment on
the same sealed side fed bm25x_growing_insert with the restated rows (the host cast over bm25x_intern, the sealed
lookup, fresh keys numbered n_terms + K + rank in key order, each row re-sorted by ordinal).  Handle arrays, info, new
keys, search rows and seals must be equal bit for bit; queries from tsvectors against the sealed side's own; refusals
that change nothing; the golden passages end to end; concurrent inserts."""
import ctypes as C
import threading

import numpy as np
import pytest

from util_cuda import free_bytes
from util_growing_tsvector import MISSING, SEED, Twin, bm_of, same_seal, same_segment
from util_index import fieldnorms, read_back
from util_lib import gpu_library, refused  # noqa: F401  (gpu_library: the module fixture m)
from util_tsvector import cast, pack_ids, pack_sorted, synthetic, word_table, write_tsvectors

pytestmark = pytest.mark.gpu


# ---- the sealed sides ----

def _words(rng, n, lo=1, hi=15):
    return list(dict.fromkeys(bytes(rng.integers(97, 123, int(rng.integers(lo, hi + 1)), dtype=np.uint8)) for _ in range(n)))


def _sealed(m, kind, rng):
    """A keyed sealed side of 400 documents over short and long words; kind: 'index' or 'sharded2' / 'sharded3'."""
    words = _words(rng, 300) + _words(rng, 60, 16, 40)
    docs = [{words[int(w)]: list(range(1, int(rng.integers(1, 4)) + 1))
             for w in rng.choice(len(words), size=int(rng.integers(1, 20)), replace=False)} for _ in range(400)]
    tsv = pack_sorted(docs)
    if kind == "index":
        return m.Index.from_tsvectors(SEED, **tsv), words
    off, keys, tf = cast(bm_of(m).intern, SEED, tsv)
    return m.ShardedIndex.from_documents(off, tf, elem_key=keys, n_shards=int(kind[-1])), words


def _batch(rng, known, fresh, n, lo=0, hi=12):
    """n tsvectors over known and fresh words (duplicates within a vector, empty vectors included)."""
    pool = known + fresh
    vs = []
    for _ in range(n):
        ln = int(rng.integers(lo, hi + 1))
        vs.append([(pool[int(w)], list(range(1, int(rng.integers(1, 4)) + 1))) for w in rng.integers(0, len(pool), ln)])
    return write_tsvectors(vs)


def _queries(rng, known, fresh, n=50):
    pool = known + fresh
    return pack_sorted([{pool[int(w)]: [1] for w in rng.integers(0, len(pool), int(rng.integers(1, 6)))}
                        for _ in range(n)])


@pytest.mark.parametrize("kind", ["index", "sharded2", "sharded3"])
@pytest.mark.parametrize("form", ["doc_len", "doc_fieldnorm"])
def test_script_equals_twin_and_seals_alike(m, orc, kind, form):
    rng = np.random.default_rng(sum(map(ord, kind + form)))
    sealed, words = _sealed(m, kind, rng)
    seg, twin = sealed.growing_segment(), Twin(m, sealed)
    fresh = _words(rng, 40, 3, 12) + _words(rng, 10, 20, 60) + [b"nul\x00inside", b"\x00", b"x" * 14 + b"\x00"]
    fresh = [w for w in fresh if w not in set(words)]
    doomed = [b"doomed-one", b"doomed-two, a lexeme long enough to be hashed"]   # every document deleted: gone at the seal
    if form == "doc_fieldnorm":    # the segment's form comes from its first insert: an ordinal one
        off, ords, tf, lens, _ = twin.rows(_batch(rng, words, [], 5))
        ords = np.where(ords >= sealed.n_terms, MISSING, ords).astype(np.uint32)   # sealed ordinals only
        twin.keys.clear()
        for s in (seg, twin.seg):
            s.insert(off, ords, tf, doc_fieldnorm=fieldnorms(orc, lens))
    for step in range(6):
        tsv = _batch(rng, words, fresh[:10 + 8 * step] if step else fresh[:5], int(rng.integers(1, 60)))
        pay = rng.integers(0, 1 << 16, (len(tsv["ent_off"]) - 1, 3)).astype(np.uint16) if step % 2 else None
        seg.insert_tsvectors(SEED, **tsv, payload=pay)
        twin.insert(orc, tsv, payload=pay, form=form)
        if step == 3:
            n0 = seg.info().n_docs
            only = write_tsvectors([[(w, [1, 2])] for w in doomed])
            seg.insert_tsvectors(SEED, **only)
            twin.insert(orc, only, form=form)
            gone = np.arange(n0, n0 + len(doomed), dtype=np.uint32)
            for s in (seg, twin.seg):
                s.delete(gone)
        if step % 2:
            dead = rng.choice(seg.info().n_docs, size=3, replace=False).astype(np.uint32)
            seg.delete(dead)
            twin.seg.delete(dead)
        same_segment(seg, twin, _queries(rng, words, fresh), f"{kind} {form} step {step}")
    # queries: the sealed side's own, with the segment's keys missing
    q = _queries(rng, words, fresh)
    q_off, q_terms = seg.tsvector_queries(SEED, **q)
    if kind == "index":
        w_off, w_terms = sealed.tsvector_queries(SEED, **q)
    else:
        off, keys, _ = cast(bm_of(m).intern, SEED, q, as_query=True)
        w_off, w_terms = off.astype(np.uint32), sealed.lookup_terms(keys)
    assert np.array_equal(q_off, w_off) and np.array_equal(q_terms, w_terms)
    qo, qk, _ = cast(bm_of(m).intern, SEED, q, as_query=True)
    own = np.array([bytes(k) in twin.keys for k in qk], bool)
    assert own.any() and (q_terms[own] == MISSING).all()
    # the seal: the segment's keys against the caller's
    dele = np.packbits((np.arange(sealed.n_docs) % 7 == 3).astype(np.uint8), bitorder="little")
    got = seg.seal(sealed_deleted=dele)
    want = twin.seg.seal(sealed_deleted=dele, new_keys=twin.new_keys())
    same_seal(got, want, f"{kind} {form} seal")
    doomed_keys = [bytes(k) for k in cast(bm_of(m).intern, SEED, write_tsvectors([[(w, [1])] for w in doomed]))[1]]
    assert all(got[3][twin.keys[k]] == MISSING for k in doomed_keys if k in twin.keys)
    assert len(got[3]) == sealed.n_terms + len(twin.keys)


def test_df0_sealed_key_and_large_batch(m, orc):
    """A lexeme equal to a sealed key with df 0 takes that ordinal; a batch of more than one cast chunk."""
    rng = np.random.default_rng(12)
    short = sorted(set(_words(rng, 200, 1, 15)))
    keys = np.zeros((len(short), 16), np.uint8)
    for i, w in enumerate(short):
        keys[i, :len(w)] = np.frombuffer(w, np.uint8)
    T = len(short)
    df0 = set(range(0, T, 9))               # terms without postings
    post_doc, post_off = [], [0]
    for t in range(T):
        docs = [] if t in df0 else sorted(rng.choice(300, size=int(rng.integers(1, 20)), replace=False).tolist())
        post_doc += docs
        post_off.append(len(post_doc))
    P = len(post_doc)
    post_tf = rng.integers(1, 4, P).astype(np.uint32)
    doc_len = np.maximum(np.bincount(post_doc, weights=post_tf, minlength=300), 1).astype(np.uint32)
    sealed = m.Index(300, doc_len, T, np.array(post_off, np.uint64), np.array(post_doc, np.uint32), post_tf,
                     term_keys=keys)
    seg, twin = sealed.growing_segment(), Twin(m, sealed)
    tsv = write_tsvectors([[(short[t], [1, 2]) for t in sorted(df0)][:5] + [(b"fresh-word", [1])]])
    seg.insert_tsvectors(SEED, **tsv)
    twin.insert(orc, tsv)
    assert len(twin.keys) == 1
    same_segment(seg, twin, tsv, "df0")
    # more than one cast chunk (2^22 entries), short and long lexemes
    big, bwords, _ = synthetic(rng, 150_000, 25, 35, 40_000, 0.02)
    assert int(big["ent_off"][-1]) > (1 << 22)
    seg.insert_tsvectors(SEED, **big)
    twin.insert(orc, big)
    same_segment(seg, twin, _queries(rng, short, bwords[:200]), "chunks")
    same_seal(seg.seal(), twin.seg.seal(new_keys=twin.new_keys()), "chunks seal")


def _expect_unchanged(seg, before, what):
    info, keys = seg.info(), seg.new_keys()
    assert (info.n_docs, info.n_deleted, info.pending) == before[0], what
    assert np.array_equal(keys, before[1]), what


def _state(seg):
    i = seg.info()
    return (i.n_docs, i.n_deleted, i.pending), seg.new_keys()


def test_refusals_change_nothing(m, orc):
    bm = bm_of(m)
    L = m.load_library()
    rng = np.random.default_rng(8)
    sealed, words = _sealed(m, "index", rng)
    # keyless index: bm25x_lookup_terms' refusal, before any device work
    kl = m.Index.from_documents(np.array([0, 2], np.uint64), np.array([1, 1], np.uint32),
                                elem_term=np.array([0, 1], np.uint32), n_terms=2)
    ks = kl.growing_segment()
    good = write_tsvectors([[(b"brand-new", [1]), (words[0], [2])], [(words[1], [1, 2])]])
    assert refused(m, lambda: ks.insert_tsvectors(SEED, **good)) == (
        1, "bm25x error 1: bm25x_lookup_terms: index was created without term keys")
    assert refused(m, lambda: ks.tsvector_queries(SEED, **good))[1].endswith("index was created without term keys")
    # caller-numbered segment: no tsvector insert
    mix = sealed.growing_segment()
    mix.insert(np.array([0, 1], np.uint64), np.array([sealed.n_terms + 2], np.uint32), np.array([1], np.uint32),
               doc_len=np.array([1], np.uint32))
    code, msg = refused(m, lambda: mix.insert_tsvectors(SEED, **good))
    assert code == 1 and "numbered by the caller" in msg
    seg = sealed.growing_segment()
    seg.tsvector_queries(SEED, **good)          # the vocabulary goes up once; nothing below may hold more memory
    seg.insert_tsvectors(SEED, **good)
    before, free = _state(seg), free_bytes()
    # an owning segment: no ordinal of its own from bm25x_growing_insert, no caller keys at the seal
    code, msg = refused(m, lambda: seg.insert(np.array([0, 1], np.uint64), np.array([sealed.n_terms], np.uint32),
                                              np.array([1], np.uint32), doc_len=np.array([1], np.uint32)))
    assert code == 1 and f"document 0 holds term ordinal {sealed.n_terms}" in msg
    seg.insert(np.array([0, 2], np.uint64), np.array([0, MISSING], np.uint32), np.array([1, 1], np.uint32),
               doc_len=np.array([2], np.uint32))
    before = _state(seg)
    code, msg = refused(m, lambda: seg.seal(new_keys=np.zeros((1, 16), np.uint8)))
    assert code == 1 and "new_keys given" in msg
    # get_new_keys below K
    n = C.c_uint32(0)
    K = len(before[1])
    assert K >= 1
    buf = np.zeros((K, 16), np.uint8)
    assert L.bm25x_growing_get_new_keys(seg.h, K - 1, bm._p(buf, C.c_uint8), C.byref(n)) == 1 and n.value == K
    assert not buf.any()
    # a merged count of 0, after the device work
    zero = pack_ids([2], *word_table([b"brand-new-2", b"zero"]), np.array([0, 1]), np.array([1, 0]))
    code, msg = refused(m, lambda: seg.insert_tsvectors(SEED, **zero))
    assert code == 1 and "sum to 0" in msg
    # a live merged tf >= 2^24: 257 entries of one sealed lexeme with 65535 positions each, plus a fresh one
    w = next(x for x in words if len(x) < 16 and sealed.lookup_terms(
        np.frombuffer(x.ljust(16, b"\0"), np.uint8).reshape(1, 16))[0] != MISSING and
        sealed.df()[sealed.lookup_terms(np.frombuffer(x.ljust(16, b"\0"), np.uint8).reshape(1, 16))[0]] > 0)
    area = w + (b"\0" if len(w) % 2 else b"") + b"\xff\xff"
    fresh = b"brand-new-3"
    area2 = area + fresh + (b"\0" if len(fresh) % 2 else b"") + b"\x01\x00"
    ents = [(0 << 12) | (len(w) << 1) | 1] * 257 + [(len(area) << 12) | (len(fresh) << 1) | 1]
    big = dict(ent_off=np.array([0, 258], np.uint64), entries=np.array(ents, np.uint32),
               byte_off=np.array([0, len(area2)], np.uint64), data=np.frombuffer(area2, np.uint8).copy())
    code, msg = refused(m, lambda: seg.insert_tsvectors(SEED, **big))
    assert code == 4 and "2^24" in msg
    _expect_unchanged(seg, before, "after refusals")
    assert free_bytes() == free


def _golden_tsvectors(golden, ids):
    docs = []
    for i in ids:
        d = {}
        for p, w in enumerate(golden["doc_lexemes"][i - 1], 1):
            d.setdefault(w.encode(), []).append(p)
        docs.append(d)
    return pack_sorted(docs)


def test_golden_end_to_end(m, orc, golden):
    """Half the passages sealed, the rest inserted as tsvectors: rows equal the twin's, the seal equals the twin's and
    finds the golden query's passages as the index built from all passages does."""
    n = len(golden["doc_lexemes"])
    half = list(range(1, n // 2 + 1))
    rest = list(range(n // 2 + 1, n + 1))
    pay = np.random.default_rng(2).integers(0, 1 << 16, (n, 3)).astype(np.uint16)
    h = len(half)
    sealed = m.Index.from_tsvectors(SEED, **_golden_tsvectors(golden, half), payload=pay[:h])
    seg, twin = sealed.growing_segment(), Twin(m, sealed)
    tsv = _golden_tsvectors(golden, rest)
    seg.insert_tsvectors(SEED, **tsv, payload=pay[h:])
    twin.insert(orc, tsv, payload=pay[h:])
    query = pack_sorted([{golden["query"].encode(): [1]}])
    same_segment(seg, twin, query, "golden")
    ix, smap, gmap, tmap = seg.seal()
    full = m.Index.from_tsvectors(SEED, **_golden_tsvectors(golden, half + rest), payload=pay)
    same_seal((ix, smap, gmap, tmap), twin.seg.seal(new_keys=twin.new_keys()), "golden seal")
    # the seal holds every passage, in id order: the query finds the passages the full build finds (a sealed survivor's
    # length is its number of postings, maintain.rs:356-360, so scores may differ from the full build's)
    assert ix.info().n_docs == full.info().n_docs == n and np.array_equal(tmap[:sealed.n_terms] != MISSING,
                                                                          np.ones(sealed.n_terms, bool))
    hits = []
    for h in (ix, full):
        q_off, q_terms = h.tsvector_queries(SEED, **query)
        r = h.search_batch(q_off, q_terms, n)
        hits.append(sorted(int(d) + 1 for d in r["doc"][0, :int(r["n"][0])]))
    assert hits[0] == hits[1] == sorted(golden["ranking_full_index"])


def test_concurrent_inserts(m, orc):
    rng = np.random.default_rng(21)
    sealed, words = _sealed(m, "index", rng)
    seg = sealed.growing_segment()
    shared = _words(rng, 30, 3, 12)
    batches = []
    for b in range(4):
        own = [w + b"-%d" % b for w in _words(rng, 10, 3, 8)]
        for j in range(3):
            batches.append(_batch(rng, words, shared + own, 40, 1, 10))
    tags = [np.tile(np.array([i, 7, 7], np.uint16), (len(t["ent_off"]) - 1, 1)) for i, t in enumerate(batches)]
    q = _queries(rng, words, shared)
    stop, errors = threading.Event(), []

    def writer(ids):
        try:
            for i in ids:
                seg.insert_tsvectors(SEED, **batches[i], payload=tags[i])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    def reader():
        try:
            while not stop.is_set():
                q_off, q_terms = seg.tsvector_queries(SEED, **q)
                seg.search_batch(q_off, q_terms, 10)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ws = [threading.Thread(target=writer, args=(list(range(3 * b, 3 * b + 3)),)) for b in range(4)]
    rd = threading.Thread(target=reader)
    rd.start()
    for t in ws:
        t.start()
    for t in ws:
        t.join()
    stop.set()
    rd.join()
    assert not errors, errors
    # each batch's ordinals are contiguous: the payload tags, in ordinal order
    seg.refresh()
    lay, der = seg.arrays()
    tag = read_back(lay, der)["payload"].reshape(-1, 3)[:, 0]
    order = [int(tag[0])]
    for i in range(1, len(tag)):
        if tag[i] != tag[i - 1]:
            order.append(int(tag[i]))
    assert sorted(order) == list(range(len(batches))), order
    # the keys: distinct, and the fresh lexemes' keys exactly
    keys = seg.new_keys()
    got = {bytes(k) for k in keys}
    assert len(got) == len(keys)
    want = set()
    for t in batches:
        _, ks, _ = cast(bm_of(m).intern, SEED, t)
        look = sealed.lookup_terms(ks)
        want |= {bytes(k) for k, o in zip(ks, look) if o == MISSING}
    assert got == want
    # the twin replaying the batches in ordinal order seals alike
    twin = Twin(m, sealed)
    for i in order:
        twin.insert(orc, batches[i], payload=tags[i])
    same_segment(seg, twin, q, "concurrent")
    same_seal(seg.seal(), twin.seg.seal(new_keys=twin.new_keys()), "concurrent seal")
