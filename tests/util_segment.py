"""The growing-segment harness: sealed indexes and the growing documents inserted into them, and the checks of a refresh
and a seal against the restatements (bm25x_growing_create and util_index for a segment's handle, bm25x_index_create and
util_maintain for a seal's result, the oracle for their searches).  growing_setup / growing_expect: one growing handle
over a synthetic sealed index and the merged rows the oracle gives for it."""
from types import SimpleNamespace

import numpy as np

from util_index import assert_matches, fieldnorms, growing_csr, read_back, restate
from util_maintain import MISSING
from util_parity import PrefixOracle, compare, live_queries, oracle_index

SEAL_KS = (1, 10, 128, 1025, 65535)
NONE = 0xFFFFFFFF
# option sets the searches of a sealed result run under: both pruning settings, every eligible query seeded, two-phase
MODES = {"prune": dict(prune=1), "no-prune": dict(prune=0),
         "seed-forced": dict(prune=1, seed_prune_min=0xFFFFFFFF, seed_dense_div=0), "twophase": dict(prune=1, twophase=1)}
DEFAULTS = dict(prune=1, seed=1, seed_prune_min=32768, seed_dense_div=64, twophase=0)


class World:
    """A sealed index and what the restatement needs of it."""

    def __init__(self, m, n_docs, off, doc, tf, doc_len, payload, keys, ix=None, k1=1.2, b=0.75):
        self.n_docs, self.n_terms = int(n_docs), len(off) - 1
        self.off, self.doc, self.tf, self.doc_len, self.payload, self.keys = off, doc, tf, doc_len, payload, keys
        self.k1, self.b = k1, b
        self.ix = ix or m.Index(n_docs, doc_len, self.n_terms, off, doc, tf, k1=k1, b=b, payload=payload, term_keys=keys)
        self.df = np.diff(off.astype(np.int64))
        self.sum_len = int(np.asarray(doc_len, np.uint64).sum())   # what a growing segment's avgdl comes from

    @staticmethod
    def from_restated(m, r, ix, k1=1.2, b=0.75):
        """The restated corpus r, whose index is the seal's result ix."""
        return World(m, r.n_docs, r.post_off, r.post_doc, r.post_tf, r.doc_len, r.payload, r.term_keys, ix, k1, b)


def random_keys(rng, n, taken=()):
    """n distinct random 16-byte keys, none in `taken`."""
    seen, out = {bytes(k) for k in taken}, []
    while len(out) < n:
        k = rng.integers(1, 256, size=16, dtype=np.uint8)
        if k.tobytes() not in seen:
            seen.add(k.tobytes())
            out.append(k)
    return np.array(out, np.uint8).reshape(-1, 16)


def sealed_docs(rng, n_docs, T):
    """Zipf-like documents ({term: tf}) over T terms, a few terms left without postings (returned, sorted), a document
    with one term at tf 3 and an empty one."""
    p = 1.0 / np.arange(1, T + 1)
    p /= p.sum()
    dead = set(rng.choice(np.arange(T // 2, T), size=4, replace=False).tolist())
    docs = []
    for d in range(n_docs):
        n = int(rng.integers(1, 20))
        terms = sorted(set(rng.choice(T, size=n, p=p).tolist()) - dead)
        docs.append({int(t): int(rng.integers(1, 6)) for t in terms})
    docs[1] = {2: 3}
    docs[2] = {}
    return docs, sorted(dead)


def sealed_world(m, orc, rng, n_docs, T, keyed, with_payload):
    """An index over sealed_docs, its lengths a few tokens above Σ tf."""
    docs, dead = sealed_docs(rng, n_docs, T)
    c = orc.Corpus.from_docs(docs, n_terms=T)
    doc_len = c.doc_len + rng.integers(0, 5, size=n_docs).astype(np.uint32)
    payload = rng.integers(0, 65536, size=(n_docs, 3)).astype(np.uint16) if with_payload else None
    keys = np.array(sorted(random_keys(rng, T).tolist()), np.uint8) if keyed else None
    return World(m, n_docs, c.post_off, c.post_doc, c.post_tf, doc_len, payload, keys), dead


class Docs:
    """Growing documents as the tests insert them, doc-major."""

    def __init__(self):
        self.off, self.term, self.tf, self.extra, self.deleted, self.payload = [0], [], [], [], [], []

    @property
    def n(self):
        return len(self.extra)

    def add(self, terms, tfs, extra, deleted, payload):
        self.term += terms
        self.tf += tfs
        self.off.append(len(self.term))
        self.extra.append(extra)
        self.deleted.append(int(deleted))
        self.payload.append(payload)

    def kw(self, orc, form, with_payload, lo=0, hi=None):
        """bm25x_growing_insert arguments of documents [lo, hi)."""
        hi = self.n if hi is None else hi
        e0, e1 = self.off[lo], self.off[hi]
        tf = np.array(self.tf[e0:e1], np.uint32)
        off = np.array(self.off[lo:hi + 1], np.uint64) - e0
        owner = np.repeat(np.arange(hi - lo), np.diff(off.astype(np.int64)))
        length = np.bincount(owner, weights=tf, minlength=hi - lo).astype(np.int64) + np.array(self.extra[lo:hi], np.int64)
        kw = dict(elem_off=off, elem_term=np.array(self.term[e0:e1], np.uint32), elem_tf=tf,
                  deleted=np.array(self.deleted[lo:hi], np.uint8))
        if form == "doc_len":
            kw["doc_len"] = length.astype(np.uint32)
        else:  # the norms the segment searches with; the seal measures Σ tf itself
            kw["doc_fieldnorm"] = fieldnorms(orc, length) if hi > lo else np.zeros(0, np.uint8)
        if with_payload:
            kw["payload"] = np.array(self.payload[lo:hi], np.uint16).reshape(-1, 3)
        return kw

    def restated(self, orc, form, with_payload, n=None, deleted=None):
        """The first n documents as util_maintain.maintain takes them (deleted: the flags at the seal)."""
        n = self.n if n is None else n
        kw = self.kw(orc, form, with_payload, 0, n)
        return SimpleNamespace(elem_off=kw["elem_off"], elem_term=kw["elem_term"], elem_tf=kw["elem_tf"],
                               deleted=np.array(self.deleted[:n] if deleted is None else deleted, np.uint8),
                               doc_len=kw.get("doc_len"), payload=kw.get("payload"))


def new_docs(rng, w, dead, docs, n, n_new, p_deleted=0.05):
    """n documents over the sealed terms (mostly), sealed terms without postings, ordinals T .. T + n_new - 1 and
    unknown tokens; an empty one now and then; tf up to 2^24 - 1."""
    T = w.n_terms
    live = np.flatnonzero(w.df > 0)
    for _ in range(n):
        k = int(rng.integers(0, 14)) if rng.random() > 0.03 else 0
        pool = set(rng.choice(live, size=k).tolist())
        if dead and rng.random() < 0.2:
            pool.add(int(rng.choice(dead)))
        if n_new and rng.random() < 0.3:
            pool.add(T + int(rng.integers(n_new)))
        terms = sorted(pool)
        tfs = rng.integers(1, 6, size=len(terms)).tolist()
        if terms and rng.random() < 0.03:
            tfs[int(rng.integers(len(tfs)))] = (1 << 24) - 1
        if rng.random() < 0.2:
            terms.append(MISSING)
            tfs.append(int(rng.integers(1, 9)))
        docs.add([int(t) for t in terms], [int(f) for f in tfs], int(rng.integers(0, 4)), rng.random() < p_deleted,
                 rng.integers(0, 65536, size=3).tolist())


def pack(bits):
    return np.packbits(np.asarray(bits, np.uint8), bitorder="little")


def check_result(m, orc, got_ix, maps, r, what, k1=1.2, b=0.75):
    """The sealed result against bm25x_index_create over the restated corpus (built with k1, b) and against the CPU
    restatement, which is returned."""
    smap, gmap, tmap = maps
    assert np.array_equal(smap, r.sealed_map), f"{what}: sealed_map"
    assert np.array_equal(gmap, r.growing_map), f"{what}: growing_map"
    assert np.array_equal(tmap, r.term_map), f"{what}: term_map"
    ref = m.Index(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf, k1=k1, b=b, payload=r.payload,
                  term_keys=r.term_keys)
    try:
        lay, der = got_ix.layout(), got_ix.derived()
        got = read_back(lay, der)
        rs = restate(orc, r.n_docs, r.post_off, r.post_doc, r.post_tf, k1, b, doc_len=r.doc_len, payload=r.payload)
        assert_matches(got, lay, der, rs, what)
        want = read_back(ref.layout(), ref.derived())
        for key in want:
            if getattr(rs, key).size:
                assert got[key].tobytes() == want[key].tobytes(), f"{what}: {key} differs from bm25x_index_create's"
        assert der.s1f_min == ref.derived().s1f_min
        a, b = got_ix.info(), ref.info()
        for f in ("n_docs", "n_terms", "n_postings", "sum_doc_len", "avgdl", "k1", "b", "n_blocks"):
            assert getattr(a, f) == getattr(b, f), f"{what}: info.{f}"
        if r.term_keys is not None and r.n_terms:
            assert np.array_equal(got_ix.lookup_terms(r.term_keys), np.arange(r.n_terms, dtype=np.uint32))
        return rs
    finally:
        ref.close()


def check_searches(orc, got_ix, r, rng, what, k1=1.2, b=0.75, ks=SEAL_KS, modes=MODES):
    """Searches on the result against the oracle's exhaustive scorer (k1, b) over the restated corpus, at every limit of
    `ks` under every option set of `modes`."""
    df = np.diff(r.post_off.astype(np.int64))
    if not (df > 0).any():
        return
    oix = orc.OracleIndex(orc.Corpus(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf, k1, b))
    po = PrefixOracle(oix, max(ks))
    q_off, q_terms = live_queries(rng, df, [1, 2, 2, 3, 3, 4, 5, 8, 12, 40][: 10 if (df > 0).sum() >= 40 else 6])
    try:
        for mode, opts in modes.items():
            for name, v in {**DEFAULTS, **opts}.items():
                got_ix.set_option(name, v)
            for k in ks:
                compare(got_ix.search_batch(q_off, q_terms, k), po, q_off, q_terms, k, what=f"{what} {mode} k={k}")
    finally:
        for name, v in DEFAULTS.items():
            got_ix.set_option(name, v)


def docs_from_postings(rng, n, term, ordinal, tf, extra_max=3):
    """Docs (arrays in place of its lists) of n growing documents holding the given postings; a length is Σ tf plus up
    to extra_max."""
    order = np.lexsort((term, ordinal))
    docs = Docs()
    docs.term, docs.tf = np.asarray(term, np.uint32)[order], np.asarray(tf, np.uint32)[order]
    docs.off = np.concatenate([[0], np.cumsum(np.bincount(ordinal, minlength=n))]).tolist()
    docs.extra = rng.integers(0, extra_max + 1, size=n)
    docs.deleted = np.zeros(n, np.uint8)
    docs.payload = rng.integers(0, 65536, size=(n, 3)).astype(np.uint16)
    return docs


def first_docs(docs, n):
    """The first n documents of docs_from_postings' Docs, sharing their deleted flags."""
    sub = Docs()
    sub.off, sub.term, sub.tf = docs.off[:n + 1], docs.term[:docs.off[n]], docs.tf[:docs.off[n]]
    sub.extra, sub.deleted, sub.payload = docs.extra[:n], docs.deleted[:n], docs.payload[:n]
    return sub


def check_segment(orc, seg, w, docs, form, with_payload, what, k1=1.2, b=0.75):
    """Every array of the segment's handle: byte-equal to bm25x_growing_create's over the same documents and flags, and to
    the CPU restatement of them with the sealed statistics of World w."""
    kw = docs.kw(orc, form, with_payload)
    ref = w.ix.growing(**kw)
    try:
        lay, der = seg.arrays()
        got = read_back(lay, der)
        g = SimpleNamespace(elem_off=kw["elem_off"], elem_term=kw["elem_term"], elem_tf=kw["elem_tf"], deleted=kw["deleted"])
        off, doc, tf = growing_csr(g, w.n_terms, w.df)
        stat = (w.n_docs, w.df, float(w.sum_len) / w.n_docs)
        if form == "doc_len":
            r = restate(orc, docs.n, off, doc, tf, k1, b, stat=stat, doc_len=kw["doc_len"], payload=kw.get("payload"))
            skip = ()
        else:   # stored norms carry no length total
            r = restate(orc, docs.n, off, doc, tf, k1, b, stat=stat, fieldnorm=kw["doc_fieldnorm"], sum_len=0,
                        payload=kw.get("payload"))
            skip = ("sum_doc_len",)
        assert_matches(got, lay, der, r, what, skip)
        want = read_back(ref.layout(), ref.derived())
        for key in want:     # an array the restatement leaves empty is one unspecified placeholder slot
            if getattr(r, key).size:
                assert got[key].tobytes() == want[key].tobytes(), f"{what}: {key} differs from bm25x_growing_create's"
        assert seg.info().n_postings == ref.info().n_postings == r.n_postings, what
        return r
    finally:
        ref.close()


def growing_setup(m, orc, seed, n_sealed, n_growing, vocab, extra_vocab, zipf):
    sealed = m.synth_corpus(seed, n_sealed, vocab, 8, 80, zipf)
    fresh = orc.Corpus.synth(seed + 1, n_growing, vocab + extra_vocab, 1, 120, zipf_s=zipf)
    deleted = (np.arange(n_growing) % 5 == 2).astype(np.uint8)
    g = orc.GrowingDocs.from_corpus(fresh, deleted)
    g.elem_term = np.where(g.elem_term >= vocab, m.TERM_MISSING, g.elem_term).astype(np.uint32)
    ix = m.Index.from_corpus(sealed)
    gix = ix.growing(g.elem_off, g.elem_term, g.elem_tf, doc_len=g.doc_len, deleted=deleted)
    return sealed, g, ix, gix, oracle_index(orc, sealed)


def growing_expect(oix, g, N, q, k, allow=None, allow_g=None):
    sd, ss, _ = oix.search_exhaustive(q, k, allow=allow)
    gd, gs = oix.search_growing(g, q, k, allow=allow_g)
    rows = sorted([(-s, int(d)) for d, s in zip(sd, ss)] + [(-s, int(d) + N) for d, s in zip(gd, gs)])[:k]
    return [d for _, d in rows], [-s for s, _ in rows]
