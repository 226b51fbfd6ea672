"""GPU: the seal of a growing segment (bm25x_growing_seal) against the restatement of maintain.rs (util_maintain): after
every seal of seeded scripts (keyless and keyed sealed indexes, both norm forms, with and without payloads, deletes in
both segments, growing tokens that are sealed terms, sealed terms with df 0, new ordinals and unknown tokens) the new
index's arrays equal byte for byte those of bm25x_index_create over the restated corpus and the CPU restatement of them,
its maps and statistics equal the restatement's, and its searches equal the oracle's exhaustive scorer on every kernel
path.  Then the edge cases, every refusal, a seal while other threads insert, delete and search, and device memory."""
import ctypes
import threading
from types import SimpleNamespace

import numpy as np
import pytest

import _pkg
from test_gpu_parity import _PrefixOracle, _compare, _live_queries
from util_cuda import cudart
from util_index import fieldnorms, read_back, restate, assert_matches
from util_maintain import MISSING, maintain

pytestmark = pytest.mark.gpu

KS = (1, 10, 128, 1025, 65535)
NONE = 0xFFFFFFFF
# option sets the searches of a sealed result run under: both pruning settings, every eligible query seeded, two-phase
MODES = {"prune": dict(prune=1), "no-prune": dict(prune=0),
         "seed-forced": dict(prune=1, seed_prune_min=0xFFFFFFFF, seed_dense_div=0), "twophase": dict(prune=1, twophase=1)}
DEFAULTS = dict(prune=1, seed=1, seed_prune_min=32768, seed_dense_div=64, twophase=0)


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


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


def _keys(rng, n, taken=()):
    """n distinct random 16-byte keys, none in `taken`."""
    seen, out = {bytes(k) for k in taken}, []
    while len(out) < n:
        k = rng.integers(1, 256, size=16, dtype=np.uint8)
        if k.tobytes() not in seen:
            seen.add(k.tobytes())
            out.append(k)
    return np.array(out, np.uint8).reshape(-1, 16)


def _sealed_docs(rng, n_docs, T):
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


def _sealed_world(m, orc, rng, n_docs, T, keyed, with_payload):
    """An index over _sealed_docs, its lengths a few tokens above Σ tf."""
    docs, dead = _sealed_docs(rng, n_docs, T)
    c = orc.Corpus.from_docs(docs, n_terms=T)
    doc_len = c.doc_len + rng.integers(0, 5, size=n_docs).astype(np.uint32)
    payload = rng.integers(0, 65536, size=(n_docs, 3)).astype(np.uint16) if with_payload else None
    keys = np.array(sorted(_keys(rng, T).tolist()), np.uint8) if keyed else None
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


def _new_docs(rng, w, dead, docs, n, n_new, p_deleted=0.05):
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


def _pack(bits):
    return np.packbits(np.asarray(bits, np.uint8), bitorder="little")


def _check_result(m, orc, got_ix, maps, r, what, k1=1.2, b=0.75):
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


def _check_searches(orc, got_ix, r, rng, what, k1=1.2, b=0.75, ks=KS, modes=MODES):
    """Searches on the result against the oracle's exhaustive scorer (k1, b) over the restated corpus, at every limit of
    `ks` under every option set of `modes`."""
    df = np.diff(r.post_off.astype(np.int64))
    if not (df > 0).any():
        return
    oix = orc.OracleIndex(orc.Corpus(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf, k1, b))
    po = _PrefixOracle(oix, max(ks))
    q_off, q_terms = _live_queries(rng, df, [1, 2, 2, 3, 3, 4, 5, 8, 12, 40][: 10 if (df > 0).sum() >= 40 else 6])
    try:
        for mode, opts in modes.items():
            for name, v in {**DEFAULTS, **opts}.items():
                got_ix.set_option(name, v)
            for k in ks:
                _compare(got_ix.search_batch(q_off, q_terms, k), po, q_off, q_terms, k, what=f"{what} {mode} k={k}")
    finally:
        for name, v in DEFAULTS.items():
            got_ix.set_option(name, v)


CASES = {("keyless", "doc_len", False): 3, ("keyless", "fieldnorm", True): 5, ("keyed", "doc_len", True): 7,
         ("keyed", "fieldnorm", False): 9}


@pytest.mark.parametrize("kind,form,with_payload", list(CASES))
def test_seal_twice_matches_maintain(m, orc, kind, form, with_payload):
    """Seal, open a segment on the result, insert and delete more, seal again: each result equals the restatement of
    maintain.rs over what it sealed (the second one: two maintains in sequence)."""
    rng = np.random.default_rng(CASES[(kind, form, with_payload)])
    keyed = kind == "keyed"
    w, dead = _sealed_world(m, orc, rng, 2500, 160, keyed, with_payload)
    n_new = 6
    new_keys = _keys(rng, n_new, w.keys) if keyed else None
    seg = w.ix.growing_segment()
    results = [w.ix]
    try:
        for round_ in range(2):
            what = f"{kind} {form} payload={with_payload} round {round_}"
            docs = Docs()
            _new_docs(rng, w, dead, docs, 150, n_new)
            seg.insert(**docs.kw(orc, form, with_payload, 0, 100))
            seg.refresh()
            seg.insert(**docs.kw(orc, form, with_payload, 100, docs.n))   # pending at the seal
            victims = rng.choice(docs.n, size=20, replace=False)
            seg.delete(victims)
            for v in victims:
                docs.deleted[int(v)] = 1
            sdel = rng.random(w.n_docs) < 0.1
            q_off, q_terms = _live_queries(rng, w.df, [1, 2, 3, 5])
            before = seg.search_batch(q_off, q_terms, 50, want_payload=True)
            info_before = seg.info()
            got = seg.seal(sealed_deleted=_pack(sdel), new_keys=new_keys)
            results.append(got[0])
            # the segment and its sealed index are unchanged: same rows, same counts
            after = seg.search_batch(q_off, q_terms, 50, want_payload=True)
            for key in ("doc", "score64", "payload", "n"):
                assert np.array_equal(before[key], after[key]), f"{what}: the old segment's rows changed ({key})"
            info_after = seg.info()
            assert (info_after.n_docs, info_after.n_deleted) == (info_before.n_docs, info_before.n_deleted)
            r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, form, with_payload), sealed_deleted=sdel,
                         sealed_payload=w.payload, sealed_keys=w.keys, new_keys=new_keys)
            _check_result(m, orc, got[0], got[1:], r, what)
            _check_searches(orc, got[0], r, rng, what)
            # the next round seals a segment opened on this result
            seg.close()
            w = World.from_restated(m, r, got[0])
            dead = np.flatnonzero(w.df == 0).tolist()
            new_keys = _keys(rng, n_new, w.keys) if keyed else None
            seg = w.ix.growing_segment()
    finally:
        seg.close()
        for ix in results:
            ix.close()


def _snapshot(seg):
    return tuple(getattr(seg.info(), f) for f, _ in type(seg.info())._fields_)


def test_edges_and_refusals(m, orc):
    rng = np.random.default_rng(41)
    w, dead = _sealed_world(m, orc, rng, 1500, 120, False, False)
    q_off, q_terms = _live_queries(rng, w.df, [1, 2, 3, 4, 6])
    seg = w.ix.growing_segment()
    made = []

    def seal_and_check(docs, sdel, what):
        got = seg.seal(sealed_deleted=_pack(sdel) if sdel is not None else None)
        made.append(got[0])
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", False), sealed_deleted=sdel)
        _check_result(m, orc, got[0], got[1:], r, what)
        _check_searches(orc, got[0], r, rng, what)
        return r

    def refused(fn, code, text):
        rows, info = seg.search_batch(q_off, q_terms, 30, want_payload=True), _snapshot(seg)
        with pytest.raises(m.Bm25xError) as e:
            fn()
        assert e.value.code == code and text in str(e.value), str(e.value)
        assert _snapshot(seg) == info
        again = seg.search_batch(q_off, q_terms, 30, want_payload=True)
        for key in ("doc", "score64", "payload", "n"):
            assert np.array_equal(rows[key], again[key]), key

    try:
        # no growing document, no delete: the postings as they were, the lengths by postings
        docs = Docs()
        r = seal_and_check(docs, None, "nothing to fold")
        assert np.array_equal(r.post_doc, w.doc) and np.array_equal(r.post_tf, w.tf)
        assert np.array_equal(r.doc_len, np.bincount(w.doc, minlength=w.n_docs).astype(np.uint32))
        # every growing document deleted
        _new_docs(rng, w, dead, docs, 80, 3)
        seg.insert(**docs.kw(orc, "doc_len", False))
        seg.delete(np.arange(docs.n))
        docs.deleted = [1] * docs.n
        seal_and_check(docs, rng.random(w.n_docs) < 0.2, "every growing document deleted")
        # every sealed document deleted
        lo = docs.n
        _new_docs(rng, w, dead, docs, 60, 3, p_deleted=0)
        seg.insert(**docs.kw(orc, "doc_len", False, lo, docs.n))
        seal_and_check(docs, np.ones(w.n_docs, bool), "every sealed document deleted")
        # everything deleted: refused
        seg.delete(np.arange(docs.n))
        docs.deleted = [1] * docs.n
        refused(lambda: seg.seal(sealed_deleted=_pack(np.ones(w.n_docs, bool))), 1, "no document survives")
        # new keys on a keyless index
        refused(lambda: seg.seal(new_keys=_keys(rng, 1)), 1, "created without term keys")
        # maps too short: refused, with the sizes a retry needs
        L = m.load_library()
        for g_cap, t_cap in ((docs.n - 1, 1 << 20), (docs.n, w.n_terms)):
            gm, tm = np.empty(max(g_cap, 1), np.uint32), np.empty(t_cap, np.uint32)
            a = m.SealArgs()
            a.growing_map, a.growing_cap = gm.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), g_cap
            a.term_map, a.term_cap = tm.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), t_cap
            h = ctypes.c_void_p()
            info = _snapshot(seg)
            assert L.bm25x_growing_seal(seg.h, ctypes.byref(a), ctypes.byref(h)) == 1 and not h.value
            assert "growing_cap" in L.bm25x_last_error().decode()
            assert a.n_growing == docs.n and a.n_source_terms == max(w.n_terms, 1 + max(t for t in docs.term if t != MISSING))
            assert _snapshot(seg) == info
    finally:
        seg.close()
        for ix in made:
            ix.close()
        w.ix.close()


def test_keyed_refusals(m, orc):
    rng = np.random.default_rng(43)
    w, dead = _sealed_world(m, orc, rng, 1200, 100, True, True)
    q_off, q_terms = _live_queries(rng, w.df, [1, 2, 3])
    seg = w.ix.growing_segment()
    try:
        docs = Docs()
        _new_docs(rng, w, dead, docs, 100, 4, p_deleted=0)
        docs.add([w.n_terms + 2], [1], 0, False, [1, 2, 3])     # ordinal T + 2 for sure
        seg.insert(**docs.kw(orc, "doc_len", True))
        rows, info = seg.search_batch(q_off, q_terms, 20, want_payload=True), _snapshot(seg)
        nk = _keys(rng, 4, w.keys)
        first = next(t for t in docs.term if w.n_terms + 2 <= t != MISSING)   # the first one inserted without a key
        cases = [(np.stack([nk[0], w.keys[17], nk[2], nk[3]]), "new key 1 equals the key of sealed term 17"),
                 (np.stack([nk[0], nk[1], nk[0], nk[3]]), "new key 0 equals new key 2"),
                 (nk[:2], f"inserted term ordinal {first} >=")]
        for keys, text in cases:
            with pytest.raises(m.Bm25xError) as e:
                seg.seal(new_keys=keys)
            assert e.value.code == 1 and text in str(e.value), str(e.value)
            assert _snapshot(seg) == info
            again = seg.search_batch(q_off, q_terms, 20, want_payload=True)
            for key in ("doc", "score64", "payload", "n"):
                assert np.array_equal(rows[key], again[key]), key
        got = seg.seal(new_keys=nk)   # and with the right keys it seals
        try:
            r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", True), sealed_payload=w.payload,
                         sealed_keys=w.keys, new_keys=nk)
            _check_result(m, orc, got[0], got[1:], r, "keyed, after the refusals")
        finally:
            got[0].close()
    finally:
        seg.close()
        w.ix.close()


def test_seal_during_inserts_deletes_and_searches(m, orc):
    """One thread inserts and deletes through a fixed script, three search the segment, the main thread seals midway.
    The seal equals the restatement of the state it reports (its ordinals; its deleted set, read off growing_map, is the
    one of a state of the script); every search returns the rows of one state of the script."""
    rng = np.random.default_rng(47)
    w, dead = _sealed_world(m, orc, rng, 2000, 140, False, False)
    q_off, q_terms = _live_queries(rng, w.df, [1, 2, 3, 4, 6, 9])
    docs = Docs()
    ops = []
    for i in range(10):
        lo = docs.n
        _new_docs(rng, w, dead, docs, int(rng.integers(20, 120)), 3)
        ops.append(("insert", lo, docs.n))
        if i % 2:
            ops.append(("delete", rng.choice(docs.n, size=15, replace=False)))
    # the states: after each op, the documents so far with their deleted flags
    states, deleted, n_now = [(0, np.zeros(0, np.uint8))], np.zeros(docs.n, np.uint8), 0
    for op in ops:
        if op[0] == "insert":
            n_now = op[2]
            deleted[op[1]:op[2]] = docs.deleted[op[1]:op[2]]
        else:
            deleted[op[1]] = 1
        states.append((n_now, deleted[:n_now].copy()))
    expect = []
    for n, dl in states:
        if n == 0:
            expect.append(w.ix.search_batch_growing(None, q_off, q_terms, 20, want_payload=True))
            continue
        kw = docs.kw(orc, "doc_len", False, 0, n)
        kw["deleted"] = dl
        ref = w.ix.growing(**kw)
        expect.append(w.ix.search_batch_growing(ref, q_off, q_terms, 20, want_payload=True))
        ref.close()
    seg = w.ix.growing_segment()
    errors, stop, sealed = [], threading.Event(), []
    started = threading.Event()

    def writer():
        try:
            for i, op in enumerate(ops):
                if op[0] == "insert":
                    seg.insert(**docs.kw(orc, "doc_len", False, op[1], op[2]))
                else:
                    seg.delete(op[1])
                if i == 2:
                    started.set()
        except Exception as e:
            errors.append(e)
        finally:
            started.set()
            stop.set()

    def reader():
        try:
            while True:
                done = stop.is_set()
                got = seg.search_batch(q_off, q_terms, 20, want_payload=True)
                assert any(all(np.array_equal(got[x], e[x]) for x in ("doc", "score", "score64", "payload", "n"))
                           for e in expect), "a search returned rows of no state of the script"
                if done:
                    break
        except Exception as e:
            errors.append(e)

    threads = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
    try:
        for t in threads:
            t.start()
        started.wait()
        sealed.append(seg.seal())
        for t in threads:
            t.join()
        assert not errors, errors[0]
        ix2, smap, gmap, tmap = sealed[0]
        n = len(gmap)
        dl = (gmap == NONE).astype(np.uint8)
        assert any(sn == n and np.array_equal(sd, dl) for sn, sd in states), "the seal took no state of the script"
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", False, n, dl))
        _check_result(m, orc, ix2, (smap, gmap, tmap), r, "concurrent seal")
    finally:
        for t in threads:
            t.join()
        seg.close()
        for s in sealed:
            s[0].close()
        w.ix.close()


def _free_bytes():
    free, total = ctypes.c_size_t(), ctypes.c_size_t()
    assert cudart().cudaMemGetInfo(ctypes.byref(free), ctypes.byref(total)) == 0
    return free.value


def test_seals_free_their_memory(m, orc):
    rng = np.random.default_rng(53)
    w, dead = _sealed_world(m, orc, rng, 1500, 120, True, False)
    docs = Docs()
    _new_docs(rng, w, dead, docs, 200, 3)
    nk = _keys(rng, 3, w.keys)

    def run(n_seal):
        seg = w.ix.growing_segment()
        seg.insert(**docs.kw(orc, "fieldnorm", False))
        for i in range(n_seal):
            seg.delete([i])
            ix, *_ = seg.seal(sealed_deleted=_pack(rng.random(w.n_docs) < 0.1), new_keys=nk)
            ix.close()
        seg.close()

    try:
        run(2)  # loads every kernel of a seal before the measurement
        free = _free_bytes()
        run(20)
        assert _free_bytes() == free, "device memory of the seal not freed"
    finally:
        w.ix.close()
