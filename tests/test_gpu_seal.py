"""GPU: the seal of a growing segment (bm25x_growing_seal) against the restatement of maintain.rs (util_maintain): after
every seal of seeded scripts (keyless and keyed sealed indexes, both norm forms, with and without payloads, deletes in
both segments, growing tokens that are sealed terms, sealed terms with df 0, new ordinals and unknown tokens) the new
index's arrays equal byte for byte those of bm25x_index_create over the restated corpus and the CPU restatement of them,
its maps and statistics equal the restatement's, and its searches equal the oracle's exhaustive scorer on every kernel
path.  Then the edge cases, every refusal, a seal while other threads insert, delete and search, and device memory."""
import ctypes
import threading

import numpy as np
import pytest

from util_cuda import free_bytes
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_maintain import MISSING, maintain
from util_parity import live_queries
from util_segment import NONE, Docs, World, check_result, check_searches, new_docs, pack, random_keys, sealed_world

pytestmark = pytest.mark.gpu

CASES = {("keyless", "doc_len", False): 3, ("keyless", "fieldnorm", True): 5, ("keyed", "doc_len", True): 7,
         ("keyed", "fieldnorm", False): 9}


@pytest.mark.parametrize("kind,form,with_payload", list(CASES))
def test_seal_twice_matches_maintain(m, orc, kind, form, with_payload):
    """Seal, open a segment on the result, insert and delete more, seal again: each result equals the restatement of
    maintain.rs over what it sealed (the second one: two maintains in sequence)."""
    rng = np.random.default_rng(CASES[(kind, form, with_payload)])
    keyed = kind == "keyed"
    w, dead = sealed_world(m, orc, rng, 2500, 160, keyed, with_payload)
    n_new = 6
    new_keys = random_keys(rng, n_new, w.keys) if keyed else None
    seg = w.ix.growing_segment()
    results = [w.ix]
    try:
        for round_ in range(2):
            what = f"{kind} {form} payload={with_payload} round {round_}"
            docs = Docs()
            new_docs(rng, w, dead, docs, 150, n_new)
            seg.insert(**docs.kw(orc, form, with_payload, 0, 100))
            seg.refresh()
            seg.insert(**docs.kw(orc, form, with_payload, 100, docs.n))   # pending at the seal
            victims = rng.choice(docs.n, size=20, replace=False)
            seg.delete(victims)
            for v in victims:
                docs.deleted[int(v)] = 1
            sdel = rng.random(w.n_docs) < 0.1
            q_off, q_terms = live_queries(rng, w.df, [1, 2, 3, 5])
            before = seg.search_batch(q_off, q_terms, 50, want_payload=True)
            info_before = seg.info()
            got = seg.seal(sealed_deleted=pack(sdel), new_keys=new_keys)
            results.append(got[0])
            # the segment and its sealed index are unchanged: same rows, same counts
            after = seg.search_batch(q_off, q_terms, 50, want_payload=True)
            for key in ("doc", "score64", "payload", "n"):
                assert np.array_equal(before[key], after[key]), f"{what}: the old segment's rows changed ({key})"
            info_after = seg.info()
            assert (info_after.n_docs, info_after.n_deleted) == (info_before.n_docs, info_before.n_deleted)
            r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, form, with_payload), sealed_deleted=sdel,
                         sealed_payload=w.payload, sealed_keys=w.keys, new_keys=new_keys)
            check_result(m, orc, got[0], got[1:], r, what)
            check_searches(orc, got[0], r, rng, what)
            # the next round seals a segment opened on this result
            seg.close()
            w = World.from_restated(m, r, got[0])
            dead = np.flatnonzero(w.df == 0).tolist()
            new_keys = random_keys(rng, n_new, w.keys) if keyed else None
            seg = w.ix.growing_segment()
    finally:
        seg.close()
        for ix in results:
            ix.close()


def _snapshot(seg):
    return tuple(getattr(seg.info(), f) for f, _ in type(seg.info())._fields_)


def test_edges_and_refusals(m, orc):
    rng = np.random.default_rng(41)
    w, dead = sealed_world(m, orc, rng, 1500, 120, False, False)
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3, 4, 6])
    seg = w.ix.growing_segment()
    made = []

    def seal_and_check(docs, sdel, what):
        got = seg.seal(sealed_deleted=pack(sdel) if sdel is not None else None)
        made.append(got[0])
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", False), sealed_deleted=sdel)
        check_result(m, orc, got[0], got[1:], r, what)
        check_searches(orc, got[0], r, rng, what)
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
        new_docs(rng, w, dead, docs, 80, 3)
        seg.insert(**docs.kw(orc, "doc_len", False))
        seg.delete(np.arange(docs.n))
        docs.deleted = [1] * docs.n
        seal_and_check(docs, rng.random(w.n_docs) < 0.2, "every growing document deleted")
        # every sealed document deleted
        lo = docs.n
        new_docs(rng, w, dead, docs, 60, 3, p_deleted=0)
        seg.insert(**docs.kw(orc, "doc_len", False, lo, docs.n))
        seal_and_check(docs, np.ones(w.n_docs, bool), "every sealed document deleted")
        # everything deleted: refused
        seg.delete(np.arange(docs.n))
        docs.deleted = [1] * docs.n
        refused(lambda: seg.seal(sealed_deleted=pack(np.ones(w.n_docs, bool))), 1, "no document survives")
        # new keys on a keyless index
        refused(lambda: seg.seal(new_keys=random_keys(rng, 1)), 1, "created without term keys")
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
    w, dead = sealed_world(m, orc, rng, 1200, 100, True, True)
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3])
    seg = w.ix.growing_segment()
    try:
        docs = Docs()
        new_docs(rng, w, dead, docs, 100, 4, p_deleted=0)
        docs.add([w.n_terms + 2], [1], 0, False, [1, 2, 3])     # ordinal T + 2 for sure
        seg.insert(**docs.kw(orc, "doc_len", True))
        rows, info = seg.search_batch(q_off, q_terms, 20, want_payload=True), _snapshot(seg)
        nk = random_keys(rng, 4, w.keys)
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
            check_result(m, orc, got[0], got[1:], r, "keyed, after the refusals")
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
    w, dead = sealed_world(m, orc, rng, 2000, 140, False, False)
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3, 4, 6, 9])
    docs = Docs()
    ops = []
    for i in range(10):
        lo = docs.n
        new_docs(rng, w, dead, docs, int(rng.integers(20, 120)), 3)
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
        check_result(m, orc, ix2, (smap, gmap, tmap), r, "concurrent seal")
    finally:
        for t in threads:
            t.join()
        seg.close()
        for s in sealed:
            s[0].close()
        w.ix.close()


def test_seals_free_their_memory(m, orc):
    rng = np.random.default_rng(53)
    w, dead = sealed_world(m, orc, rng, 1500, 120, True, False)
    docs = Docs()
    new_docs(rng, w, dead, docs, 200, 3)
    nk = random_keys(rng, 3, w.keys)

    def run(n_seal):
        seg = w.ix.growing_segment()
        seg.insert(**docs.kw(orc, "fieldnorm", False))
        for i in range(n_seal):
            seg.delete([i])
            ix, *_ = seg.seal(sealed_deleted=pack(rng.random(w.n_docs) < 0.1), new_keys=nk)
            ix.close()
        seg.close()

    try:
        run(2)  # loads every kernel of a seal before the measurement
        free = free_bytes()
        run(20)
        assert free_bytes() == free, "device memory of the seal not freed"
    finally:
        w.ix.close()
