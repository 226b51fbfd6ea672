"""GPU: the growing segment over a document-sharded index (bm25x_growing_open_sharded, bm25x_growing_seal_sharded).

Every case runs beside a twin: an unsharded index over the same corpus whose own segment receives the same inserts,
deletes and refreshes.  After every step the sharded segment's rows (all five arrays) and its `queries` / `postings`
equal the twin's, and its growing handle equals the twin's byte for byte, at 1..16 shards with default and adversarial
bounds, every limit and the four option sets of util_segment.MODES.  Its seal equals, shard by shard and byte for byte,
bm25x_sharded_create over the restatement of maintain.rs (util_maintain) with the bounds the layout rule gives, its maps
equal the restatement's and the twin's seal's, and its rows equal those of the twin's sealed index.  Then the layout
edges, the refusals, a seal while other threads insert, delete and search, device memory and two devices."""
import ctypes
import threading

import numpy as np
import pytest

from util_cuda import free_bytes
from util_index import read_back
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_maintain import MISSING, maintain
from util_parity import ROWS, live_queries, same_rows
from util_segment import DEFAULTS, MODES, NONE, SEAL_KS, Docs, World, new_docs, pack, random_keys, sealed_world

pytestmark = pytest.mark.gpu



def _bounds(kind, S, n_docs):
    """Shard bounds: None (balanced by postings) or adversarial: one-document shards first, one large shard, and a
    one-document LAST shard (the growing documents follow a single sealed one)."""
    if kind == "default" or S == 1:
        return None
    return np.array([0] + [1 + i for i in range(S - 2)] + [n_docs - 1, n_docs], np.uint32)


def _sharded(m, w, S, bounds, devices=None):
    return m.ShardedIndex(w.n_docs, w.doc_len, w.n_terms, w.off, w.doc, w.tf, payload=w.payload, term_keys=w.keys,
                          n_shards=S, doc_bounds=bounds, devices=devices)


def _set_options(handles, opts):
    for h in handles:
        for name, v in {**DEFAULTS, **opts}.items():
            h.set_option(name, v)


def _same_arrays(a, b, what):
    """Two index handles' arrays ((IndexLayout, IndexDerived) pairs), byte for byte, scalars included."""
    (la, da), (lb, db) = a, b
    for f, _ in type(la)._fields_:
        if f not in ("dev_ptr", "device"):
            assert np.array_equal(np.asarray(getattr(la, f)), np.asarray(getattr(lb, f))), f"{what}: layout.{f}"
    assert (da.n_champ, da.s1f_min) == (db.n_champ, db.s1f_min), f"{what}: derived scalars"
    ga, gb = read_back(la, da), read_back(lb, db)
    for key in ga:
        if key in ("blk", "blk_ub") and la.n_blocks == 0 or key == "champ" and da.n_champ == 0:
            continue  # one placeholder slot of unspecified content
        assert ga[key].tobytes() == gb[key].tobytes(), f"{what}: {key} differs"


def _search_pair(seg, twin, rng, w, q_off, q_terms, k, what, allow=True):
    """The sharded segment against its twin at limit k, with and without the two prefilters."""
    n_g = seg.info().n_docs
    runs = [(None, None)]
    if allow:
        runs.append((pack(rng.random(w.n_docs) < 0.7), pack(rng.random(max(n_g, 1)) < 0.7)))
    for al, ag in runs:
        a = seg.search_batch(q_off, q_terms, k, allow=al, allow_growing=ag, allow_growing_docs=max(n_g - 3, 0),
                             want_payload=True)
        b = twin.search_batch(q_off, q_terms, k, allow=al, allow_growing=ag, allow_growing_docs=max(n_g - 3, 0),
                              want_payload=True)
        same_rows(a, b, f"{what} allow={al is not None}")
        assert (a["stats"].queries, a["stats"].postings) == (b["stats"].queries, b["stats"].postings), what


PARITY = [(S, kind) for S in (1, 2, 3, 8, 16) for kind in ("default", "adversarial") if S > 1 or kind == "default"]


@pytest.mark.parametrize("k", SEAL_KS)
@pytest.mark.parametrize("S,kind", PARITY)
def test_search_parity(m, orc, S, kind, k):
    """Seeded scripts of inserts, deletes and refreshes; after every step the rows under every option set, and the growing
    handle's arrays, equal the twin's.  S = 16 with k = 65535 merges 17 lists."""
    seed = 1000 * S + 10 * SEAL_KS.index(k) + (kind == "adversarial")
    rng = np.random.default_rng(seed)
    form = ("doc_len", "fieldnorm")[seed % 2]
    with_payload = bool(seed // 2 % 2)
    keyed = bool(seed // 4 % 2)
    w, dead = sealed_world(m, orc, rng, 600, 90, keyed, with_payload)
    sx = _sharded(m, w, S, _bounds(kind, S, w.n_docs))
    seg, twin = sx.growing_segment(), w.ix.growing_segment()
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 2, 3, 4, 5, 8, 12, 40])
    what = f"S={S} {kind} k={k} {form} payload={with_payload} keyed={keyed}"
    try:
        # before the first insert: the sharded search itself, stats included
        a = seg.search_batch(q_off, q_terms, k, want_payload=True)
        b = sx.search_batch(q_off, q_terms, k, want_payload=True)
        same_rows(a, b, f"{what} empty")
        for f in ("queries", "postings", "postings_fetched", "launches", "bytes_algo"):
            assert getattr(a["stats"], f) == getattr(b["stats"], f), f"{what} empty: stats.{f}"
        assert seg.info().device == 0
        docs = Docs()
        for step in range(3):
            lo = docs.n
            new_docs(rng, w, dead, docs, int(rng.integers(20, 90)), 4, p_deleted=0.1)
            kw = docs.kw(orc, form, with_payload, lo, docs.n)
            seg.insert(**kw)
            twin.insert(**kw)
            if step == 1:
                seg.refresh()
                twin.refresh()
            victims = rng.choice(docs.n, size=min(docs.n, 6), replace=False)
            seg.delete(victims)
            twin.delete(victims)
            for mode, opts in MODES.items():
                _set_options((sx, w.ix), opts)
                _search_pair(seg, twin, rng, w, q_off, q_terms, k, f"{what} step {step} {mode}", allow=mode == "prune")
            _set_options((sx, w.ix), {})
            _same_arrays(seg.arrays(), twin.arrays(), f"{what} step {step}: growing handle")
            a, b = seg.info(), twin.info()
            assert (a.n_docs, a.n_deleted, a.n_postings, a.pending) == (b.n_docs, b.n_deleted, b.n_postings, b.pending)
    finally:
        seg.close()
        twin.close()
        sx.close()
        w.ix.close()


def _new_bounds(old_bounds, sdel, n_growing_kept):
    """The layout rule: per old shard its survivors, the last one plus the growing survivors; empty shards dropped."""
    kept = [int((~sdel[old_bounds[s]:old_bounds[s + 1]]).sum()) for s in range(len(old_bounds) - 1)]
    kept[-1] += n_growing_kept
    keep = [s for s in range(len(kept)) if kept[s]]
    return np.concatenate([[0], np.cumsum([kept[s] for s in keep])]).astype(np.uint32), keep


def _check_sealed(m, orc, got, twin_got, r, old_bounds, sdel, old_devices, rng, what, ks=SEAL_KS, modes=MODES):
    """The sharded seal `got` (ShardedIndex, maps) against bm25x_sharded_create over the restated corpus r with the
    layout rule's bounds and devices, against the restatement's maps and the twin's, and its rows against the twin's
    sealed index."""
    sx, smap, gmap, tmap = got
    tix, tsmap, tgmap, ttmap = twin_got
    for name, a, b, c in (("sealed_map", smap, r.sealed_map, tsmap), ("growing_map", gmap, r.growing_map, tgmap),
                          ("term_map", tmap, r.term_map, ttmap)):
        assert np.array_equal(a, b) and np.array_equal(a, c), f"{what}: {name}"
    bounds, keep = _new_bounds(old_bounds, sdel, int((r.growing_map != NONE).sum()))
    assert np.array_equal(sx.doc_bounds(), bounds), f"{what}: bounds {sx.doc_bounds()} != {bounds}"
    devices = [old_devices[s] for s in keep]
    ref = m.ShardedIndex(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf, payload=r.payload,
                         term_keys=r.term_keys, n_shards=len(bounds) - 1, doc_bounds=bounds, devices=devices)
    try:
        for j in range(len(bounds) - 1):
            got_j = sx.shard_arrays(j)
            assert got_j[0].device == devices[j], f"{what}: shard {j} device"
            _same_arrays(got_j, ref.shard_arrays(j), f"{what}: shard {j}")
        a, b = sx.info(), ref.info()
        for f in ("n_docs", "n_terms", "n_postings", "sum_doc_len", "avgdl", "k1", "b", "n_blocks", "device_bytes",
                  "device"):
            assert getattr(a, f) == getattr(b, f), f"{what}: info.{f}"
        if r.term_keys is not None and r.n_terms:
            assert np.array_equal(sx.lookup_terms(r.term_keys), np.arange(r.n_terms, dtype=np.uint32))
    finally:
        ref.close()
    df = np.diff(r.post_off.astype(np.int64))
    if not (df > 0).any():
        return
    q_off, q_terms = live_queries(rng, df, [1, 2, 2, 3, 4, 5, 8, 12, 40][: 9 if (df > 0).sum() >= 40 else 5])
    try:
        for mode, opts in modes.items():
            _set_options((sx, tix), opts)
            for k in ks:
                same_rows(sx.search_batch(q_off, q_terms, k, want_payload=True),
                           tix.search_batch(q_off, q_terms, k, want_payload=True), f"{what} {mode} k={k}")
    finally:
        _set_options((sx, tix), {})


SEALS = {("keyless", "doc_len", False, 2): 3, ("keyless", "fieldnorm", True, 3): 5, ("keyed", "doc_len", True, 3): 7,
         ("keyed", "fieldnorm", False, 2): 9}


@pytest.mark.parametrize("kind,form,with_payload,S", list(SEALS))
def test_seal_matches_restatement(m, orc, kind, form, with_payload, S):
    """Seal after a script, then open a segment on the result, insert and delete more, seal again: every result equals
    the restatement, shard by shard, and the twin's seal."""
    rng = np.random.default_rng(SEALS[(kind, form, with_payload, S)])
    keyed = kind == "keyed"
    w, dead = sealed_world(m, orc, rng, 1500, 140, keyed, with_payload)
    sx = _sharded(m, w, S, None)
    made = [sx, w.ix]
    seg = twin = None
    try:
        for round_ in range(2):
            what = f"{kind} {form} payload={with_payload} S={S} round {round_}"
            old_bounds = sx.doc_bounds()
            seg, twin = sx.growing_segment(), w.ix.growing_segment()
            docs = Docs()
            new_docs(rng, w, dead, docs, 120, 5)
            for lo, hi in ((0, 70), (70, docs.n)):
                kw = docs.kw(orc, form, with_payload, lo, hi)
                seg.insert(**kw)
                twin.insert(**kw)
                if lo == 0:
                    seg.refresh()
                    twin.refresh()
            victims = rng.choice(docs.n, size=15, replace=False)
            seg.delete(victims)
            twin.delete(victims)
            for v in victims:
                docs.deleted[int(v)] = 1
            sdel = rng.random(w.n_docs) < 0.1
            new_keys = random_keys(rng, 5, w.keys) if keyed else None
            q_off, q_terms = live_queries(rng, w.df, [1, 2, 3, 5])
            before = seg.search_batch(q_off, q_terms, 40, want_payload=True)
            got = seg.seal(sealed_deleted=pack(sdel), new_keys=new_keys)
            made.append(got[0])
            twin_got = twin.seal(sealed_deleted=pack(sdel), new_keys=new_keys)
            made.append(twin_got[0])
            same_rows(before, seg.search_batch(q_off, q_terms, 40, want_payload=True), f"{what}: the old segment")
            r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, form, with_payload), sealed_deleted=sdel,
                         sealed_payload=w.payload, sealed_keys=w.keys, new_keys=new_keys)
            _check_sealed(m, orc, got, twin_got, r, old_bounds, sdel, [0] * (len(old_bounds) - 1), rng, what)
            seg.close()
            twin.close()
            seg = twin = None
            sx, w = got[0], World.from_restated(m, r, twin_got[0])
            dead = np.flatnonzero(w.df == 0).tolist()
    finally:
        for s in (seg, twin):
            if s is not None:
                s.close()
        for h in made:
            h.close()


@pytest.mark.parametrize("case", ["first", "middle", "last-with-growing", "last-without-growing", "compaction",
                                  "sixteen"])
def test_layout_edges(m, orc, case):
    """Every sealed document of one shard deleted (the first, a middle one, the last with and without growing
    survivors), a seal with no insert, and a 16-shard index."""
    rng = np.random.default_rng(61 + len(case))
    w, dead = sealed_world(m, orc, rng, 800, 100, False, True)
    S = 16 if case == "sixteen" else 4
    bounds = np.array([0, 150, 400, 650, 800], np.uint32) if S == 4 else None
    sx = _sharded(m, w, S, bounds)
    old_bounds = sx.doc_bounds()
    seg, twin = sx.growing_segment(), w.ix.growing_segment()
    made = [sx, w.ix]
    try:
        docs = Docs()
        if case != "compaction":
            new_docs(rng, w, dead, docs, 60, 3)
            seg.insert(**docs.kw(orc, "doc_len", True))
            twin.insert(**docs.kw(orc, "doc_len", True))
        if case == "last-without-growing":
            seg.delete(np.arange(docs.n))
            twin.delete(np.arange(docs.n))
            docs.deleted = [1] * docs.n
        sdel = rng.random(w.n_docs) < 0.05
        s = {"first": 0, "middle": 2, "last-with-growing": 3, "last-without-growing": 3}.get(case)
        if s is not None:
            sdel[old_bounds[s]:old_bounds[s + 1]] = True
        got = seg.seal(sealed_deleted=pack(sdel))
        made.append(got[0])
        twin_got = twin.seal(sealed_deleted=pack(sdel))
        made.append(twin_got[0])
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", True), sealed_deleted=sdel,
                     sealed_payload=w.payload)
        _check_sealed(m, orc, got, twin_got, r, old_bounds, sdel, [0] * S, rng, case, ks=(1, 10, 1025))
        n_shards = len(got[0].doc_bounds()) - 1
        assert n_shards == S - (case in ("first", "middle", "last-without-growing")), n_shards
    finally:
        seg.close()
        twin.close()
        for h in made:
            h.close()


def _snapshot(seg):
    return tuple(getattr(seg.info(), f) for f, _ in type(seg.info())._fields_)


def test_refusals(m, orc):
    """bm25x_growing_seal's refusals with their codes and messages, named by bm25x_growing_seal_sharded; the cross-kind
    refusals; nothing changes on a refusal."""
    rng = np.random.default_rng(67)
    w, dead = sealed_world(m, orc, rng, 900, 100, True, True)
    sx = _sharded(m, w, 3, None)
    seg, plain = sx.growing_segment(), w.ix.growing_segment()
    L = m.load_library()
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3])
    try:
        docs = Docs()
        new_docs(rng, w, dead, docs, 80, 4, p_deleted=0)
        docs.add([w.n_terms + 2], [1], 0, False, [1, 2, 3])     # ordinal T + 2 for sure
        seg.insert(**docs.kw(orc, "doc_len", True))
        plain.insert(**docs.kw(orc, "doc_len", True))
        rows, info = seg.search_batch(q_off, q_terms, 20, want_payload=True), _snapshot(seg)
        nk = random_keys(rng, 4, w.keys)

        def refused(fn, code, text):
            with pytest.raises(m.Bm25xError) as e:
                fn()
            assert e.value.code == code and text in str(e.value), str(e.value)
            assert _snapshot(seg) == info
            same_rows(rows, seg.search_batch(q_off, q_terms, 20, want_payload=True), text)

        first = next(t for t in docs.term if w.n_terms + 2 <= t != MISSING)
        who = "bm25x_growing_seal_sharded: "
        refused(lambda: seg.seal(new_keys=np.stack([nk[0], w.keys[17], nk[2], nk[3]])), 1,
                who + "new key 1 equals the key of sealed term 17")
        refused(lambda: seg.seal(new_keys=np.stack([nk[0], nk[1], nk[0], nk[3]])), 1, who + "new key 0 equals new key 2")
        refused(lambda: seg.seal(new_keys=nk[:2]), 1, who + f"inserted term ordinal {first} >=")
        seg.delete(np.arange(docs.n))
        rows, info = seg.search_batch(q_off, q_terms, 20, want_payload=True), _snapshot(seg)
        refused(lambda: seg.seal(new_keys=nk, sealed_deleted=pack(np.ones(w.n_docs, bool))), 1,
                who + "no document survives")
        # maps too short: refused with the sizes a retry needs
        for g_cap, t_cap in ((docs.n - 1, 1 << 20), (docs.n, w.n_terms)):
            gm, tm = np.empty(max(g_cap, 1), np.uint32), np.empty(t_cap, np.uint32)
            a = m.SealArgs()
            a.new_keys, a.n_new_keys = nk.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), len(nk)
            a.growing_map, a.growing_cap = gm.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), g_cap
            a.term_map, a.term_cap = tm.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), t_cap
            h = ctypes.c_void_p()
            assert L.bm25x_growing_seal_sharded(seg.h, ctypes.byref(a), ctypes.byref(h)) == 1 and not h.value
            assert L.bm25x_last_error().decode().startswith(who + "growing_cap=")
            assert (a.n_growing, a.n_source_terms) == (docs.n, w.n_terms + len(nk))
            assert _snapshot(seg) == info
        # a surviving posting with tf >= 2^24 (only the dormant list can hold one: the handle refuses it at insert)
        seg2 = sx.growing_segment()
        try:
            dead_term = dead[0]
            seg2.insert(elem_off=np.array([0, 1], np.uint64), elem_term=np.array([dead_term], np.uint32),
                        elem_tf=np.array([1 << 24], np.uint32), doc_len=np.array([5], np.uint32))
            with pytest.raises(m.Bm25xError) as e:
                seg2.seal(new_keys=nk)
            assert e.value.code == 4 and (who + "term frequency >= 2^24") in str(e.value), str(e.value)
        finally:
            seg2.close()
        # the cross-kind calls
        h = ctypes.c_void_p()
        assert L.bm25x_growing_seal(seg.h, ctypes.byref(m.SealArgs()), ctypes.byref(h)) == 1 and not h.value
        msg = L.bm25x_last_error().decode()
        assert msg.startswith("bm25x_growing_seal: ") and "bm25x_growing_seal_sharded" in msg, msg
        assert L.bm25x_growing_seal_sharded(plain.h, ctypes.byref(m.SealArgs()), ctypes.byref(h)) == 1 and not h.value
        msg = L.bm25x_last_error().decode()
        assert msg.startswith(who) and msg.endswith("with bm25x_growing_seal"), msg
        assert _snapshot(seg) == info
        same_rows(rows, seg.search_batch(q_off, q_terms, 20, want_payload=True), "after the cross-kind refusals")
    finally:
        seg.close()
        plain.close()
        sx.close()
        w.ix.close()


def test_seal_during_inserts_deletes_and_searches(m, orc):
    """One thread inserts and deletes through a fixed script, three search the segment, the main thread seals midway:
    the seal equals the restatement of the state it reports (n_growing ordinals, the deleted set read off growing_map),
    and every search succeeds with the rows of one state of the script."""
    rng = np.random.default_rng(71)
    w, dead = sealed_world(m, orc, rng, 1500, 120, False, False)
    sx = _sharded(m, w, 3, None)
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3, 4, 6, 9])
    docs = Docs()
    ops = []
    for i in range(8):
        lo = docs.n
        new_docs(rng, w, dead, docs, int(rng.integers(20, 100)), 3)
        ops.append(("insert", lo, docs.n))
        if i % 2:
            ops.append(("delete", rng.choice(docs.n, size=12, replace=False)))
    # the rows of every state, from the twin's unsharded segment stepped through the script
    twin = w.ix.growing_segment()
    expect = [twin.search_batch(q_off, q_terms, 20, want_payload=True)]
    for op in ops:
        if op[0] == "insert":
            twin.insert(**docs.kw(orc, "doc_len", False, op[1], op[2]))
        else:
            twin.delete(op[1])
        expect.append(twin.search_batch(q_off, q_terms, 20, want_payload=True))
    twin.close()
    seg = sx.growing_segment()
    errors, stop, started, sealed = [], threading.Event(), threading.Event(), []

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
                assert any(all(np.array_equal(got[x], e[x]) for x in ROWS) for e in expect), \
                    "a search returned rows of no state of the script"
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
        nsx, smap, gmap, tmap = sealed[0]
        n = len(gmap)
        dl = (gmap == NONE).astype(np.uint8)
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", False, n, dl))
        assert np.array_equal(smap, r.sealed_map) and np.array_equal(tmap, r.term_map)
        bounds, _ = _new_bounds(sx.doc_bounds(), np.zeros(w.n_docs, bool), int((gmap != NONE).sum()))
        ref = m.ShardedIndex(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf, payload=r.payload,
                             n_shards=len(bounds) - 1, doc_bounds=bounds)
        try:
            assert np.array_equal(nsx.doc_bounds(), bounds)
            for j in range(len(bounds) - 1):
                _same_arrays(nsx.shard_arrays(j), ref.shard_arrays(j), f"concurrent seal: shard {j}")
        finally:
            ref.close()
    finally:
        for t in threads:
            t.join()
        seg.close()
        for s in sealed:
            s[0].close()
        sx.close()
        w.ix.close()


def test_seals_free_their_memory(m, orc):
    rng = np.random.default_rng(73)
    w, dead = sealed_world(m, orc, rng, 1200, 110, True, False)
    sx = _sharded(m, w, 3, None)
    docs = Docs()
    new_docs(rng, w, dead, docs, 150, 3)
    nk = random_keys(rng, 3, w.keys)
    q_off, q_terms = live_queries(rng, w.df, [1, 2, 3])

    def run(n_seal):
        seg = sx.growing_segment()
        seg.insert(**docs.kw(orc, "fieldnorm", False))
        for i in range(n_seal):
            seg.delete([i])
            seg.search_batch(q_off, q_terms, 10)
            nsx, *_ = seg.seal(sealed_deleted=pack(rng.random(w.n_docs) < 0.1), new_keys=nk)
            nsx.close()
        seg.close()

    try:
        run(2)  # loads every kernel of a seal before the measurement
        free = free_bytes()
        run(15)
        assert free_bytes() == free, "device memory of the sharded seal not freed"
    finally:
        sx.close()
        w.ix.close()


def test_two_devices(m, orc):
    """Shards on devices [0, 1, 1]: the growing handle on device 1, the merge on device 0; the seal keeps the devices."""
    if m.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    rng = np.random.default_rng(79)
    w, dead = sealed_world(m, orc, rng, 900, 100, False, True)
    sx = _sharded(m, w, 3, None, devices=[0, 1, 1])
    old_bounds = sx.doc_bounds()
    seg, twin = sx.growing_segment(), w.ix.growing_segment()
    made = [sx, w.ix]
    try:
        docs = Docs()
        new_docs(rng, w, dead, docs, 80, 3)
        seg.insert(**docs.kw(orc, "doc_len", True))
        twin.insert(**docs.kw(orc, "doc_len", True))
        assert seg.info().device == 1
        q_off, q_terms = live_queries(rng, w.df, [1, 2, 3, 5, 8])
        for k in (1, 10, 1025):
            _search_pair(seg, twin, rng, w, q_off, q_terms, k, f"two devices k={k}")
        _same_arrays(seg.arrays(), twin.arrays(), "two devices: growing handle")
        sdel = rng.random(w.n_docs) < 0.1
        got = seg.seal(sealed_deleted=pack(sdel))
        made.append(got[0])
        twin_got = twin.seal(sealed_deleted=pack(sdel))
        made.append(twin_got[0])
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", True), sealed_deleted=sdel,
                     sealed_payload=w.payload)
        _check_sealed(m, orc, got, twin_got, r, old_bounds, sdel, [0, 1, 1], rng, "two devices", ks=(1, 10, 1025))
    finally:
        seg.close()
        twin.close()
        for h in made:
            h.close()
