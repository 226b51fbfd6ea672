"""GPU: the rebind of a growing segment to the index its seal built (bm25x_growing_rebind / _sharded).  In each scenario
documents A are inserted, the segment is sealed (its snapshot: A), documents B are inserted, some of A and B deleted,
and the segment rebound.  The rebound segment then equals, array for array, field for field and row for row, a fresh
segment on the new index fed the restatement of the carried documents (util_rebind); its late deletes are the
restatement's.  Then owned keys, a lifecycle of several rounds, every refusal, threads across the rebind, an empty
carry and device memory."""
import threading
import time
from types import SimpleNamespace

import numpy as np
import pytest

from util_cuda import free_bytes
from util_index import DERIVED, LAYOUT, read_back
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_maintain import MISSING, maintain
from util_parity import live_queries
from util_rebind import insert_kw, late_deleted, restate
from util_segment import (MODES, DEFAULTS, Docs, World, check_result, growing_expect, new_docs, random_keys,
                          sealed_world)
from util_tsvector import pack_sorted

pytestmark = pytest.mark.gpu

ROWS = ("doc", "score", "score64", "payload", "n")
SEED = bytes((5 * i + 11) & 0xFF for i in range(32))


def _sharded(m, w, S=3):
    return m.ShardedIndex(w.n_docs, w.doc_len, w.n_terms, w.off, w.doc, w.tf, payload=w.payload, term_keys=w.keys,
                          n_shards=S)


def same_segment(seg, ref, what):
    """Arrays of both handles byte for byte (an array of at most 8 bytes on both may be an unspecified placeholder), and
    every field of get_info."""
    a, b = seg.info(), ref.info()
    for f, _ in type(a)._fields_:
        assert getattr(a, f) == getattr(b, f), f"{what}: info.{f} {getattr(a, f)} != {getattr(b, f)}"
    if not a.n_docs:
        return
    (la, da), (lb, db) = seg.arrays(), ref.arrays()
    for f in ("n_docs", "n_terms", "n_postings", "n_postings_padded", "n_blocks", "sum_doc_len", "k1", "b", "avgdl"):
        assert getattr(la, f) == getattr(lb, f), f"{what}: layout.{f}"
    assert da.n_champ == db.n_champ and da.s1f_min == db.s1f_min, what
    got, want = read_back(la, da), read_back(lb, db)
    for name, _ in LAYOUT + DERIVED:
        if got[name].nbytes <= 8 and want[name].nbytes <= 8:
            continue
        assert got[name].tobytes() == want[name].tobytes(), f"{what}: {name} differs from the fresh segment's"


def same_rows(seg, ref, side, df, rng, what, modes=MODES, ks=(1, 10, 128, 1025)):
    """Every search of seg equals ref's, on every kernel path and limit (queries over the terms of df > 0)."""
    if not (df > 0).any():
        return
    q_off, q_terms = live_queries(rng, df, [1, 2, 3, 4, 6])
    try:
        for mode, opts in modes.items():
            for name, v in {**DEFAULTS, **opts}.items():
                side.set_option(name, v)
            for k in ks:
                a, b = seg.search_batch(q_off, q_terms, k, want_payload=True), ref.search_batch(q_off, q_terms, k,
                                                                                              want_payload=True)
                for key in ROWS:
                    assert np.array_equal(a[key], b[key]), f"{what} {mode} k={k}: {key}"
    finally:
        for name, v in DEFAULTS.items():
            side.set_option(name, v)


def oracle_rows(orc, r_seal, r, seg, rng, what, k1=1.2, b=0.75):
    """The rebound segment's rows against the oracle: the exhaustive scan of the new sealed corpus (r_seal) and of the
    carried documents (r) with the new sealed statistics (search.rs:49-135)."""
    df = np.diff(r_seal.post_off.astype(np.int64))
    if not (df > 0).any():
        return
    oix = orc.OracleIndex(orc.Corpus(r_seal.n_docs, r_seal.doc_len, r_seal.n_terms, r_seal.post_off, r_seal.post_doc,
                                     r_seal.post_tf, k1, b))
    g = None
    n_carried = len(r.elem_off) - 1
    if n_carried:
        # tokens the new sealed segment lacks never match (search.rs:60-62): MISSING for the oracle, still last per row
        term = np.where(r.elem_term >= r_seal.n_terms, MISSING, r.elem_term).astype(np.uint32)
        dl = r.doc_len if r.doc_len is not None else np.zeros(n_carried, np.uint32)
        g = orc.GrowingDocs(r.elem_off, term, r.elem_tf, dl, r.deleted)
        if r.doc_len is None:
            g.fieldnorm = np.ascontiguousarray(r.doc_fieldnorm, np.uint8)
    q_off, q_terms = live_queries(rng, df, [1, 2, 3, 5])
    res = seg.search_batch(q_off, q_terms, 10)
    for i in range(len(q_off) - 1):
        q = q_terms[q_off[i]:q_off[i + 1]]
        if g is None:
            sd, ss, _ = oix.search_exhaustive(q, 10)
            ed, es = [int(d) for d in sd], [float(x) for x in ss]
        else:
            ed, es = growing_expect(oix, g, r_seal.n_docs, q, 10)
        n = int(res["n"][i])
        assert res["doc"][i, :n].tolist() == ed and res["score64"][i, :n].tolist() == es, f"{what}: oracle q{i}"


def carried_docs(docs, r, n_folded):
    """The carried documents r as Docs, ordinal i of the rebound segment as document i."""
    nxt = Docs()
    off = r.elem_off.astype(np.int64)
    for i in range(len(off) - 1):
        nxt.add([int(t) for t in r.elem_term[off[i]:off[i + 1]]], [int(f) for f in r.elem_tf[off[i]:off[i + 1]]],
                docs.extra[n_folded + i], r.deleted[i], r.payload[i].tolist())
    return nxt


def old_docs(orc, docs, form, with_payload):
    kw = docs.kw(orc, form, with_payload)
    return SimpleNamespace(elem_off=kw["elem_off"], elem_term=kw["elem_term"], elem_tf=kw["elem_tf"],
                           deleted=np.array(docs.deleted, np.uint8), payload=kw.get("payload"), doc_len=kw.get("doc_len"),
                           doc_fieldnorm=kw.get("doc_fieldnorm"))


def keep_terms(docs, lo, keep):
    """Documents [lo, n) of docs without the elements whose term fails keep(t) (MISSING always stays)."""
    off, term, tf = docs.off[:lo + 1], docs.term[:docs.off[lo]], docs.tf[:docs.off[lo]]
    for d in range(lo, docs.n):
        for t, f in zip(docs.term[docs.off[d]:docs.off[d + 1]], docs.tf[docs.off[d]:docs.off[d + 1]]):
            if t == MISSING or keep(t):
                term.append(t)
                tf.append(f)
        off.append(len(term))
    docs.off, docs.term, docs.tf = off, term, tf


def round_trip(m, orc, rng, w, side, seg, docs, dead, form, with_payload, keyed, n_a, n_b, what, sdel=None):
    """Insert A, seal, insert B, delete some of A and B, rebind; check against the restatement.  Returns the new index,
    the restatement of the seal (util_maintain) and the late deletes."""
    lo = docs.n
    new_docs(rng, w, dead, docs, n_a, 6)
    seg.insert(**docs.kw(orc, form, with_payload, lo, docs.n))
    nk = random_keys(rng, 6, w.keys) if keyed else None
    ix2, smap, gmap, tmap = seg.seal(sealed_deleted=None if sdel is None else np.packbits(sdel, bitorder="little"),
                                     new_keys=nk)
    n_folded = docs.n
    r_seal = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, form, with_payload), sealed_deleted=sdel,
                      sealed_payload=w.payload, sealed_keys=w.keys, new_keys=nk)
    new_docs(rng, w, dead, docs, n_b, 10 if not keyed else 6)
    if keyed:   # B holds only ordinals the seal gave keys to (the others are refused: test_refusals)
        keep_terms(docs, n_folded, lambda t: t < len(tmap) and tmap[t] != MISSING)
    seg.insert(**docs.kw(orc, form, with_payload, n_folded, docs.n))
    victims = rng.choice(docs.n, size=min(docs.n, 25), replace=False)
    seg.delete(victims)
    for v in victims:
        docs.deleted[int(v)] = 1
    late = seg.rebind(ix2)
    assert seg.sealed is ix2
    r = restate(old_docs(orc, docs, form, with_payload), n_folded, "caller" if keyed else "keyless", term_map=tmap)
    assert np.array_equal(late, late_deleted(gmap, docs.deleted)), what
    ref = ix2.growing_segment()
    try:
        if r.elem_off.size > 1:
            ref.insert(**insert_kw(r))
            ref.refresh()
        same_segment(seg, ref, what)
        same_rows(seg, ref, ix2, np.diff(r_seal.post_off.astype(np.int64)), rng, what)
        oracle_rows(orc, r_seal, r, seg, rng, what)
    finally:
        ref.close()
    return ix2, r_seal, late, carried_docs(docs, r, n_folded)


CASES = [(kind, form, pay, sh) for kind in ("keyless", "keyed") for form in ("doc_len", "fieldnorm")
         for pay in (False, True) for sh in (False, True)]


@pytest.mark.parametrize("kind,form,with_payload,sharded", CASES)
def test_rebind_matches_a_fresh_segment(m, orc, kind, form, with_payload, sharded):
    rng = np.random.default_rng(100 + CASES.index((kind, form, with_payload, sharded)))
    keyed = kind == "keyed"
    w, dead = sealed_world(m, orc, rng, 700, 80, keyed, with_payload)
    side = _sharded(m, w) if sharded else w.ix
    seg = side.growing_segment()
    made = []
    try:
        docs = Docs()
        ix2, *_ = round_trip(m, orc, rng, w, side, seg, docs, dead, form, with_payload, keyed, 150, 60,
                             f"{kind} {form} payload={with_payload} sharded={sharded}",
                             sdel=rng.random(w.n_docs) < 0.1)
        made.append(ix2)
        if sharded:
            side.close()
    finally:
        seg.close()
        for ix in made:
            ix.close()
        w.ix.close()


def test_lifecycle_three_rounds(m, orc):
    """Three rounds of insert, seal, insert, delete, rebind on a keyless index: after each rebind the segment equals its
    restatement, and each seal equals util_maintain over the previous one, applied in sequence to the whole history."""
    rng = np.random.default_rng(71)
    w, dead = sealed_world(m, orc, rng, 900, 90, False, True)
    seg = w.ix.growing_segment()
    made = [w.ix]
    docs = Docs()
    late = np.zeros(0, np.uint32)
    try:
        for rnd in range(3):
            # the late deletes of the last rebind are sealed documents deleted before this seal
            sdel = rng.random(w.n_docs) < 0.08
            sdel[late] = True
            ix2, r_seal, late, docs = round_trip(m, orc, rng, w, w.ix, seg, docs, dead, "doc_len", True, False, 120, 50,
                                                 f"round {rnd}", sdel=sdel)
            made.append(ix2)
            check_result(m, orc, ix2, (r_seal.sealed_map, r_seal.growing_map, r_seal.term_map), r_seal, f"round {rnd}")
            w = World.from_restated(m, r_seal, ix2)
            dead = np.flatnonzero(w.df == 0).tolist()
        # a last seal of what the rounds left, with the last late deletes, equals the restatement
        sdel = np.zeros(w.n_docs, bool)
        sdel[late] = True
        got = seg.seal(sealed_deleted=np.packbits(sdel, bitorder="little"))
        made.append(got[0])
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", True), sealed_deleted=sdel,
                     sealed_payload=w.payload)
        check_result(m, orc, got[0], got[1:], r, "final seal")
    finally:
        seg.close()
        for ix in made:
            ix.close()


def _snapshot(seg):
    return tuple(getattr(seg.info(), f) for f, _ in type(seg.info())._fields_)


def test_refusals(m, orc):
    rng = np.random.default_rng(73)
    w, dead = sealed_world(m, orc, rng, 600, 70, True, False)
    seg = w.ix.growing_segment()
    sx = _sharded(m, w, 2)
    sseg = sx.growing_segment()
    made = []
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3])

    def refused(fn, text, s=seg):
        s.refresh()
        rows, info = s.search_batch(q_off, q_terms, 20, want_payload=True), _snapshot(s)
        arrays = read_back(*s.arrays()) if info[0] else None
        with pytest.raises(m.Bm25xError) as e:
            fn()
        assert e.value.code == 1 and text in str(e.value), str(e.value)
        assert _snapshot(s) == info
        if arrays is not None:
            again = read_back(*s.arrays())
            assert all(arrays[k].tobytes() == again[k].tobytes() for k in arrays if arrays[k].nbytes > 8)
        rows2 = s.search_batch(q_off, q_terms, 20, want_payload=True)
        assert all(np.array_equal(rows[k], rows2[k]) for k in ROWS)

    try:
        docs = Docs()
        new_docs(rng, w, dead, docs, 80, 0, p_deleted=0)
        seg.insert(**docs.kw(orc, "doc_len", False))
        refused(lambda: seg.rebind(w.ix), "no seal to rebind to")
        foreign = m.Index(w.n_docs, w.doc_len, w.n_terms, w.off, w.doc, w.tf, term_keys=w.keys)
        made.append(foreign)
        first = seg.seal()
        made.append(first[0])
        refused(lambda: seg.rebind(foreign), "not the one the segment's latest seal returned")
        second = seg.seal()
        made.append(second[0])
        refused(lambda: seg.rebind(first[0]), "not the one the segment's latest seal returned")
        # a destroyed result's address may come back with the next handle: the serial tells them apart
        third = seg.seal()
        third[0].close()
        again = [m.Index(w.n_docs, w.doc_len, w.n_terms, w.off, w.doc, w.tf, term_keys=w.keys) for _ in range(3)]
        made.extend(again)
        for ix in again:
            refused(lambda: seg.rebind(ix), "not the one the segment's latest seal returned")
        # the kind, both ways
        L = m.load_library()
        bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
        a = m.RebindArgs()
        sseg.insert(**docs.kw(orc, "doc_len", False))
        ss = sseg.seal()
        made.append(ss[0])
        refused(lambda: bm._check(L.bm25x_growing_rebind_sharded(seg.h, ss[0].h, bm.C.byref(a))),
                "opened over an unsharded index")
        refused(lambda: bm._check(L.bm25x_growing_rebind(sseg.h, second[0].h, bm.C.byref(a))),
                "opened over a document-sharded index", s=sseg)
        # keyed caller-numbered: an ordinal the seal had no key for, and one whose key vanished
        fourth = seg.seal()
        made.append(fourth[0])
        n0 = docs.n
        docs.add([w.n_terms + 3], [2], 0, False, [1, 2, 3])
        seg.insert(**docs.kw(orc, "doc_len", False, n0, docs.n))
        refused(lambda: seg.rebind(fourth[0]), f"growing ordinal {n0} holds term ordinal {w.n_terms + 3} >= n_source_terms")
        seg.delete([n0])
        docs.deleted[n0] = 1
        late = seg.rebind(fourth[0])   # the refused document deleted: the rebind goes through
        assert late.size == 0
        # a new key whose only document was deleted before the seal vanishes; a carried document holding it is refused
        T4 = fourth[0].n_terms
        one = dict(elem_off=np.array([0, 1], np.uint64), elem_term=np.array([T4], np.uint32),
                   elem_tf=np.array([1], np.uint32), doc_len=np.array([3], np.uint32))
        n1 = seg.info().n_docs
        seg.insert(**one, deleted=np.array([1], np.uint8))
        ix5, _, gmap, tmap = seg.seal(new_keys=random_keys(rng, 1, w.keys))
        made.append(ix5)
        assert tmap[T4] == MISSING
        seg.insert(**one)
        refused(lambda: seg.rebind(ix5), f"growing ordinal {n1 + 1} holds term ordinal {T4}, whose key vanished")
        seg.delete([n1 + 1])
        seg.rebind(ix5)
        sseg.rebind(ss[0])
    finally:
        seg.close()
        sseg.close()
        sx.close()
        for ix in made:
            ix.close()
        w.ix.close()


def test_owned_keys(m, orc):
    """Tsvector inserts: keys of B the seal folded in, keys only deleted A documents held (vanished, renumbered), keys new
    after the seal and sealed keys the seal dropped; the rebound segment against insert_tsvectors of B into a fresh
    segment (the same payloads, the same deletes)."""
    words = [f"w{i}".encode() for i in range(30)]
    sealed = [{words[i % 30]: [1], words[(3 * i) % 30]: [2, 3]} for i in range(60)]
    sealed[0] = {b"dropme": [1], words[0]: [1]}        # the only sealed holder of "dropme": deleted at the seal
    ix = m.Index.from_tsvectors(SEED, **pack_sorted(sealed))
    seg = ix.growing_segment()
    made = [ix]
    try:
        a_docs = [{b"new1": [1], words[1]: [1]}, {b"gone": [1], words[2]: [2]}, {b"new2": [1, 2]}, {words[5]: [1]}]
        pay_a = np.arange(12, dtype=np.uint16).reshape(4, 3)
        seg.insert_tsvectors(SEED, **pack_sorted(a_docs), payload=pay_a)
        seg.delete([1])                                 # "gone" was held by deleted A document 1 only
        sdel = np.zeros(ix.n_docs, bool)
        sdel[0] = True
        ix2, smap, gmap, tmap = seg.seal(sealed_deleted=np.packbits(sdel, bitorder="little"))
        made.append(ix2)
        b_docs = [{b"new1": [1], b"fresh": [2]}, {b"gone": [1], b"dropme": [2], words[7]: [1]},
                  {b"new2": [1], b"zzz": [1, 2]}, {words[3]: [4], b"fresh": [1]}]
        pay_b = np.arange(100, 112, dtype=np.uint16).reshape(4, 3)
        seg.insert_tsvectors(SEED, **pack_sorted(b_docs), payload=pay_b)
        seg.delete([0, 3])                              # A documents, after the snapshot
        late = seg.rebind(ix2)
        assert late.tolist() == sorted(int(gmap[o]) for o in (0, 3))
        ref = ix2.growing_segment()
        try:
            ref.insert_tsvectors(SEED, **pack_sorted(b_docs), payload=pay_b)
            ref.refresh()
            assert seg.new_keys().tobytes() == ref.new_keys().tobytes()
            assert len(seg.new_keys()) == 4                # dropme, fresh, gone, zzz
            same_segment(seg, ref, "owned keys")
            q_off, q_terms = seg.tsvector_queries(SEED, **pack_sorted([{b"new1": [1]}, {b"fresh": [1], words[7]: [1]}]))
            q2 = ref.tsvector_queries(SEED, **pack_sorted([{b"new1": [1]}, {b"fresh": [1], words[7]: [1]}]))
            assert np.array_equal(q_off, q2[0]) and np.array_equal(q_terms, q2[1])
            for k in (1, 10):
                a, b = seg.search_batch(q_off, q_terms, k, want_payload=True), ref.search_batch(q_off, q_terms, k,
                                                                                               want_payload=True)
                assert all(np.array_equal(a[x], b[x]) for x in ROWS)
            # and the next seal of both is the same index
            s1, s2 = seg.seal(), ref.seal()
            made += [s1[0], s2[0]]
            assert all(np.array_equal(x, y) for x, y in zip(s1[1:], s2[1:]))
            g1, g2 = read_back(s1[0].layout(), s1[0].derived()), read_back(s2[0].layout(), s2[0].derived())
            assert all(g1[k].tobytes() == g2[k].tobytes() for k in g1 if g1[k].nbytes > 8)
        finally:
            ref.close()
    finally:
        seg.close()
        for x in made:
            x.close()


def test_threads_across_the_rebind(m, orc):
    """Searches run while the seal and the rebind run: every row set is the pre- or the post-rebind one.  The old index
    is destroyed right after rebind returns."""
    rng = np.random.default_rng(79)
    w, dead = sealed_world(m, orc, rng, 1200, 100, False, False)
    seg = w.ix.growing_segment()
    docs = Docs()
    new_docs(rng, w, dead, docs, 200, 4)
    seg.insert(**docs.kw(orc, "doc_len", False))
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3, 5])
    ix2, *_ = seg.seal()
    n_folded = docs.n
    new_docs(rng, w, dead, docs, 40, 4)
    seg.insert(**docs.kw(orc, "doc_len", False, n_folded, docs.n))
    pre = seg.search_batch(q_off, q_terms, 20, want_payload=True)
    r = restate(old_docs(orc, docs, "doc_len", False), n_folded, "keyless")
    ref = ix2.growing_segment()
    ref.insert(**insert_kw(r))
    post = ref.search_batch(q_off, q_terms, 20, want_payload=True)
    errors, stop = [], threading.Event()

    def reader():
        try:
            while not stop.is_set():
                got = seg.search_batch(q_off, q_terms, 20, want_payload=True)
                assert any(all(np.array_equal(got[x], e[x]) for x in ROWS) for e in (pre, post)), "rows of no binding"
        except Exception as e:
            errors.append(e)

    threads = [threading.Thread(target=reader) for _ in range(3)]
    try:
        for t in threads:
            t.start()
        seg.rebind(ix2)
        w.ix.close()                    # the old index, right after the rebind returned
        for _ in range(5):
            got = seg.search_batch(q_off, q_terms, 20, want_payload=True)
            assert all(np.array_equal(got[x], post[x]) for x in ROWS)
        stop.set()
        for t in threads:
            t.join()
        assert not errors, errors[0]
        same_segment(seg, ref, "after the threads")
    finally:
        stop.set()
        for t in threads:
            t.join()
        ref.close()
        seg.close()
        ix2.close()


def test_empty_carry(m, orc):
    """Nothing inserted after the snapshot: no handle, and searches and stats are bm25x_search_batch's on the new index."""
    rng = np.random.default_rng(83)
    w, dead = sealed_world(m, orc, rng, 600, 60, False, False)
    seg = w.ix.growing_segment()
    docs = Docs()
    new_docs(rng, w, dead, docs, 100, 3)
    seg.insert(**docs.kw(orc, "doc_len", False))
    ix2, *_ = seg.seal()
    try:
        seg.delete([0, 1])
        late = seg.rebind(ix2)
        assert seg.info().n_docs == 0 and seg.info().n_postings == 0 and seg.info().device_bytes == 0
        assert late.size == sum(1 for o in (0, 1) if not docs.deleted[o])
        q_off, q_terms = live_queries(rng, np.ones(ix2.n_terms, np.int64), [1, 2, 3])
        a, b = seg.search_batch(q_off, q_terms, 30, want_payload=True), ix2.search_batch(q_off, q_terms, 30,
                                                                                         want_payload=True)
        for x in ("doc", "score", "score64", "n"):
            assert np.array_equal(a[x], b[x]), x
        assert a["stats"].queries == b["stats"].queries
    finally:
        seg.close()
        ix2.close()
        w.ix.close()


def test_rebinds_free_their_memory(m, orc):
    rng = np.random.default_rng(89)
    w, dead = sealed_world(m, orc, rng, 800, 80, False, False)
    docs = Docs()
    new_docs(rng, w, dead, docs, 120, 3)

    def run(n):
        seg = w.ix.growing_segment()
        side = w.ix
        for i in range(n):
            seg.insert(**docs.kw(orc, "fieldnorm", False))
            ix2, *_ = seg.seal()
            seg.insert(**docs.kw(orc, "fieldnorm", False, 0, 30))
            seg.delete([i])
            seg.rebind(ix2)
            if side is not w.ix:
                side.close()
            side = ix2
        seg.close()
        if side is not w.ix:
            side.close()

    try:
        run(2)
        free = free_bytes()
        run(8)
        assert free_bytes() == free, "device memory of the rebind not freed"
    finally:
        w.ix.close()


def _rows_well_formed(got, k, n_ids):
    for i in range(len(got["n"])):
        n = int(got["n"][i])
        assert n <= k and (got["doc"][i, :n] < n_ids).all(), "a row out of range"
        assert (np.diff(got["score64"][i, :n]) <= 0).all(), "a row out of order"


def test_writers_across_seal_and_rebind(m, orc):
    """One thread inserts through a fixed script (tsvectors, and by ordinal documents whose every token is unknown, some
    of them deleted), three search and cast queries, and the main thread seals, rebinds and closes the old index midway.
    Every row is well formed.  Then the rebound segment equals a fresh segment on the new index fed the documents after
    the seal's snapshot in commit order: the same handle arrays, info and rows, the same owned keys (up to their
    numbering, which depends on how the documents were batched), and the same next seal."""
    rng = np.random.default_rng(97)
    words = [f"w{i}".encode() for i in range(60)]
    sealed = [{words[int(i)]: [1] for i in rng.choice(60, size=5, replace=False)} for _ in range(400)]
    ix = m.Index.from_tsvectors(SEED, **pack_sorted(sealed))
    n_sealed = ix.n_docs
    seg = ix.growing_segment()
    ops, pay = [], 0
    for i in range(30):
        n = int(rng.integers(5, 25))
        payload = (np.arange(pay, pay + n)[:, None] * np.array([1, 3, 7]) % 65536).astype(np.uint16)
        pay += n
        if i % 3 == 2:
            tf = rng.integers(1, 5, size=n).astype(np.uint32)
            ops.append(("ordinal", dict(elem_off=np.arange(n + 1, dtype=np.uint64),
                                        elem_term=np.full(n, MISSING, np.uint32), elem_tf=tf,
                                        doc_len=tf + rng.integers(0, 3, size=n).astype(np.uint32), payload=payload,
                                        deleted=(rng.random(n) < 0.3).astype(np.uint8))))
        else:
            docs = []
            for _ in range(n):
                d = {words[int(j)]: [1] for j in rng.choice(60, size=int(rng.integers(1, 6)), replace=False)}
                if rng.random() < 0.4:
                    d[f"new{int(rng.integers(40))}".encode()] = [1, 2]
                docs.append(d)
            ops.append(("tsv", docs, payload))
    qdocs = [{words[1]: [1], words[2]: [1]}, {words[3]: [1], b"new3": [1]}, {b"new7": [1]}]
    q_off, q_terms = ix.tsvector_queries(SEED, **pack_sorted(qdocs))
    errors, stop, halfway = [], threading.Event(), threading.Event()

    def write(s, op):
        if op[0] == "ordinal":
            s.insert(**op[1])
        else:
            s.insert_tsvectors(SEED, **pack_sorted(op[1]), payload=op[2])

    def writer():
        try:
            for i, op in enumerate(ops):
                write(seg, op)
                if i == 10:
                    halfway.set()
        except Exception as e:
            errors.append(e)
        finally:
            halfway.set()

    def reader():
        try:
            while not stop.is_set():
                got = seg.search_batch(q_off, q_terms, 10, want_payload=True)
                _rows_well_formed(got, 10, 1 << 31)
                seg.tsvector_queries(SEED, **pack_sorted(qdocs))
        except Exception as e:
            errors.append(e)

    threads = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
    made = []
    try:
        for t in threads:
            t.start()
        halfway.wait()
        ix2, smap, gmap, tmap = seg.seal()
        made.append(ix2)
        late = seg.rebind(ix2)
        ix.close()                       # the old index, right after the rebind returned
        assert late.size == 0            # no folded document was deleted after the snapshot
        threads[0].join()
        stop.set()
        for t in threads:
            t.join()
        assert not errors, errors[0]
        # the documents in commit order, those after the snapshot replayed on a fresh segment
        n_folded, at, ref = len(gmap), 0, ix2.growing_segment()
        try:
            for op in ops:
                n = len(op[1]) if op[0] == "tsv" else len(op[1]["doc_len"])
                lo = max(n_folded - at, 0)
                at += n
                if lo >= n:
                    continue
                if op[0] == "tsv":
                    ref.insert_tsvectors(SEED, **pack_sorted(op[1][lo:]), payload=op[2][lo:])
                else:
                    kw = op[1]
                    ref.insert(elem_off=kw["elem_off"][lo:] - kw["elem_off"][lo], elem_term=kw["elem_term"][lo:],
                               elem_tf=kw["elem_tf"][lo:], doc_len=kw["doc_len"][lo:], payload=kw["payload"][lo:],
                               deleted=kw["deleted"][lo:])
            assert seg.info().n_docs == at - n_folded
            seg.refresh()
            ref.refresh()
            same_segment(seg, ref, "writers")
            ka, kb = seg.new_keys(), ref.new_keys()
            assert sorted(map(bytes, ka)) == sorted(map(bytes, kb))
            qa, qb = seg.tsvector_queries(SEED, **pack_sorted(qdocs)), ref.tsvector_queries(SEED, **pack_sorted(qdocs))
            assert np.array_equal(qa[0], qb[0]) and np.array_equal(qa[1], qb[1])
            for k in (1, 10, 100):
                a, b = (x.search_batch(qa[0], qa[1], k, want_payload=True) for x in (seg, ref))
                assert all(np.array_equal(a[x], b[x]) for x in ROWS), k
            s1, s2 = seg.seal(), ref.seal()
            made += [s1[0], s2[0]]
            assert np.array_equal(s1[1], s2[1]) and np.array_equal(s1[2], s2[2])
            g1, g2 = read_back(s1[0].layout(), s1[0].derived()), read_back(s2[0].layout(), s2[0].derived())
            assert all(g1[x].tobytes() == g2[x].tobytes() for x in g1 if g1[x].nbytes > 8)
        finally:
            ref.close()
        assert n_sealed > 0
    finally:
        stop.set()
        halfway.set()
        for t in threads:
            t.join()
        seg.close()
        for x in made:
            x.close()


def _overlap(m, seg, earlier, seal_kw, delay):
    """A seal in a thread of its own and, `delay` seconds after it started, the rebind to `earlier`: (whether the rebind
    went through, the seal's result or the message of its refusal)."""
    out = {}

    def sealer():
        try:
            out["seal"] = seg.seal(**seal_kw)
        except m.Bm25xError as e:
            out["seal"] = str(e)

    t = threading.Thread(target=sealer)
    t.start()
    time.sleep(delay)
    try:
        seg.rebind(earlier)
        rebound = True
    except m.Bm25xError as e:
        assert "not the one the segment's latest seal returned" in str(e), str(e)
        rebound = False
    t.join()
    return rebound, out["seal"]


def test_seal_that_a_rebind_overtakes_before_its_snapshot_is_refused(m, orc):
    """The seal takes the binding, then spends a long time on its keys before its snapshot; a rebind lands meanwhile.
    The seal is refused ('seal it again') and the rebind carries exactly what it should."""
    rng = np.random.default_rng(101)
    w, dead = sealed_world(m, orc, rng, 600, 70, True, False)
    seg = w.ix.growing_segment()
    made = []
    try:
        docs = Docs()
        new_docs(rng, w, dead, docs, 100, 0)
        seg.insert(**docs.kw(orc, "doc_len", False))
        ix1, _, gmap, tmap = seg.seal()
        made.append(ix1)
        n_folded = docs.n
        new_docs(rng, w, dead, docs, 40, 0, p_deleted=0)
        seg.insert(**docs.kw(orc, "doc_len", False, n_folded, docs.n))
        many = rng.integers(0, 256, size=(3_000_000, 16), dtype=np.uint8)   # sorted and checked before the snapshot
        rebound, res = _overlap(m, seg, ix1, dict(new_keys=many), 0.1)
        assert rebound
        assert isinstance(res, str) and "seal it again" in res, res
        r = restate(old_docs(orc, docs, "doc_len", False), n_folded, "caller", term_map=tmap)
        ref = ix1.growing_segment()
        try:
            ref.insert(**insert_kw(r))
            ref.refresh()
            same_segment(seg, ref, "after the refused seal")
        finally:
            ref.close()
        with pytest.raises(m.Bm25xError, match="no seal to rebind to"):
            seg.rebind(ix1)
    finally:
        seg.close()
        for x in made:
            x.close()
        w.ix.close()


def test_seal_that_a_rebind_overtakes_after_its_snapshot_records_nothing(m, orc):
    """A seal of a large index takes its snapshot, then builds; a rebind to the earlier seal lands meanwhile.  The seal
    returns its index but records nothing: a rebind to it is refused ('no seal to rebind to'), since its n_growing counts
    ordinals the segment no longer has.  Each attempt runs with another delay until that order is met; every other order
    met on the way must be consistent (the seal refused before its snapshot; or the seal first, the earlier result
    refused; or the seal after the rebind, over the rebound ordinals)."""
    rng = np.random.default_rng(103)
    c = m.synth_corpus(0xB25C0DE0 + 5, 4_000_000, 50_000, 48, 80, 0.0)
    ix = m.Index.from_corpus(c)
    c.free()
    seg = ix.growing_segment()
    side, made, seen = ix, [], set()

    def batch(n):
        tf = rng.integers(1, 5, size=(n, 4)).astype(np.uint32)
        term = np.sort(rng.choice(50_000, size=(n, 4)), axis=1).astype(np.uint32)
        term[:, 1:] += np.cumsum(np.diff(term, axis=1) == 0, axis=1).astype(np.uint32)   # strictly ascending
        return dict(elem_off=np.arange(0, 4 * n + 1, 4, dtype=np.uint64), elem_term=term.ravel(), elem_tf=tf.ravel(),
                    doc_len=tf.sum(axis=1).astype(np.uint32) + 2)

    try:
        for delay in (0.04, 0.02, 0.07, 0.1, 0.01, 0.15):
            seg.insert(**batch(1000))
            earlier, *_ = seg.seal()
            seg.insert(**batch(200))
            before = seg.info().n_docs
            rebound, res = _overlap(m, seg, earlier, {}, delay)
            after = seg.info().n_docs
            if rebound:
                made.append(side)
                side = earlier
            else:
                made.append(earlier)
            if isinstance(res, str):
                assert rebound and "seal it again" in res, res
                seen.add("refused")
                continue
            new, _, gmap2, _ = res
            try:
                late = seg.rebind(new)
            except m.Bm25xError as e:
                assert rebound and "no seal to rebind to" in str(e), str(e)
                assert len(gmap2) == before       # its snapshot was of the ordinals before the rebind
                seen.add("no record")
                made.append(new)
                break
            # accepted: the seal's ordinals are those of the binding the rebind left
            assert late.size == 0
            assert len(gmap2) == (after if rebound else before), (len(gmap2), before, after)
            assert seg.info().n_docs == (after if rebound else before) - len(gmap2)
            seen.add("after" if rebound else "before")
            made.append(side)
            side = new
        assert "no record" in seen, seen
    finally:
        seg.close()
        made.append(side)
        for x in made:
            if x is not None:
                x.close()
