"""GPU: the mutable growing segment (bm25x_growing_*) against bm25x_growing_create + bm25x_search_batch_growing on the
same documents, bit for bit, after every step of a seeded script of inserts, deletes and refreshes: every array of the
segment's handle (the 13 of the layout, the doc-id copy and the champion lists), every output of its searches, its
statistics, its refusals, concurrent searches while another thread inserts and deletes, and its device memory."""
import threading

import numpy as np
import pytest

from util_cuda import free_bytes
from util_index import CHAMP_L, assert_matches, fieldnorms, growing_csr, read_back, restate
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import oracle_index, query_csr, same_rows
from util_segment import growing_expect

pytestmark = pytest.mark.gpu

TF_MAX = (1 << 24) - 1
KS = (1, 10, 128, 129, 224, 1024, 1025, 65535)


@pytest.fixture(scope="module")
def world(m, orc):
    sealed = m.synth_corpus(0x5E6, 6000, 400, 8, 60, 0.8)
    ix = m.Index.from_corpus(sealed)
    sd = orc.GrowingDocs.from_corpus(orc.Corpus(sealed.n_docs, sealed.doc_len, sealed.n_terms, sealed.post_off,
                                                sealed.post_doc, sealed.post_tf))
    yield dict(sealed=sealed, ix=ix, sdocs=sd, oix=oracle_index(orc, sealed))
    ix.close()


class Docs:
    """Growing documents, doc-major, as the tests accumulate them."""

    def __init__(self):
        self.off, self.term, self.tf, self.len, self.deleted, self.payload = [0], [], [], [], [], []

    @property
    def n(self):
        return len(self.len)

    def add(self, terms, tfs, deleted, payload):
        self.term += list(terms)
        self.tf += list(tfs)
        self.off.append(len(self.term))
        self.len.append(int(sum(tfs)) if len(tfs) else 1)
        self.deleted.append(int(deleted))
        self.payload.append(payload)

    def arrays(self, lo=0, hi=None):
        hi = self.n if hi is None else hi
        off = np.array(self.off[lo:hi + 1], np.uint64) - self.off[lo]
        e0, e1 = self.off[lo], self.off[hi]
        return dict(elem_off=off, elem_term=np.array(self.term[e0:e1], np.uint32),
                    elem_tf=np.array(self.tf[e0:e1], np.uint32), doc_len=np.array(self.len[lo:hi], np.uint32),
                    deleted=np.array(self.deleted[lo:hi], np.uint8),
                    payload=np.array(self.payload[lo:hi], np.uint16).reshape(-1, 3))


def _new_docs(rng, w, docs, n, p_deleted=0.05):
    """n documents: random terms of the sealed vocabulary and beyond it (raw ordinals >= n_terms and TERM_MISSING),
    tf = 2^24 - 1 now and then, some deleted on insert, every tenth a copy of a sealed document (ties across segments)."""
    T = w["sealed"].n_terms
    sd = w["sdocs"]
    for _ in range(n):
        if rng.random() < 0.1:
            d = int(rng.integers(sd.n_docs))
            e0, e1 = int(sd.elem_off[d]), int(sd.elem_off[d + 1])
            terms, tfs = sd.elem_term[e0:e1].tolist(), sd.elem_tf[e0:e1].tolist()
        else:
            terms = sorted(rng.choice(T + 30, size=int(rng.integers(1, 40)), replace=False).tolist())
            tfs = rng.integers(1, 6, size=len(terms)).tolist()
            if rng.random() < 0.05:
                tfs[int(rng.integers(len(tfs)))] = TF_MAX
            terms = [t if t < T + 15 else 0xFFFFFFFF for t in terms]   # unknown tokens (ascending check skips them)
        docs.add(terms, tfs, rng.random() < p_deleted, rng.integers(0, 65535, size=3).tolist())


def _kw(docs, form, with_payload, lo=0, hi=None, orc=None):
    a = docs.arrays(lo, hi)
    kw = dict(elem_off=a["elem_off"], elem_term=a["elem_term"], elem_tf=a["elem_tf"], deleted=a["deleted"])
    if form == "doc_len":
        kw["doc_len"] = a["doc_len"]
    else:
        kw["doc_fieldnorm"] = fieldnorms(orc, a["doc_len"]) if len(a["doc_len"]) else np.zeros(0, np.uint8)
    if with_payload:
        kw["payload"] = a["payload"]
    return kw


def _reference(w, docs, form, with_payload, orc):
    """bm25x_growing_create over every document inserted so far, with their deleted flags."""
    kw = _kw(docs, form, with_payload, orc=orc)
    return w["ix"].growing(**kw)


def _same_arrays(seg, ref, w, docs, form, with_payload, orc, what):
    lay, der = seg.arrays()
    got = read_back(lay, der)
    ix, sealed = w["ix"], w["sealed"]
    a = docs.arrays()
    sdf = ix.df()
    g = orc.GrowingDocs(a["elem_off"], a["elem_term"], a["elem_tf"], a["doc_len"], a["deleted"])
    off, doc, tf = growing_csr(g, sealed.n_terms, sdf)
    stat = (sealed.n_docs, sdf, float(int(sealed.doc_len.astype(np.uint64).sum())) / sealed.n_docs)
    pay = a["payload"] if with_payload else None
    if form == "doc_len":
        r = restate(orc, docs.n, off, doc, tf, 1.2, 0.75, stat=stat, doc_len=a["doc_len"], payload=pay)
        skip = ()
    else:
        r = restate(orc, docs.n, off, doc, tf, 1.2, 0.75, stat=stat, fieldnorm=fieldnorms(orc, a["doc_len"]), sum_len=0,
                    payload=pay)
        skip = ("sum_doc_len",)
    assert_matches(got, lay, der, r, what, skip)
    # byte-equal to bm25x_growing_create's arrays, but for the placeholder slot of an array the restatement leaves empty
    # (blk and blk_ub of a handle without postings): its content is unspecified
    want = read_back(ref.layout(), ref.derived())
    for key in want:
        if getattr(r, key).size:
            assert got[key].tobytes() == want[key].tobytes(), f"{what}: {key} differs from bm25x_growing_create's"
    return r


def _queries(rng, T, nq, lo=1, hi=8):
    qs = [sorted(rng.choice(T, size=int(rng.integers(lo, hi + 1)), replace=False).tolist()) for _ in range(nq)]
    qs.append([3, 3, 7, 0xFFFFFFFF, T + 5])                              # duplicate and missing terms
    qs.append(sorted(rng.choice(T, size=40, replace=False).tolist()))    # 33..64 live terms: two passes
    qs.append([])
    return query_csr(qs)


def _search_both(seg, ix, ref, q_off, q_terms, k, allow=None, allow_g=None, allow_g_docs=None):
    got = seg.search_batch(q_off, q_terms, k, allow=allow, allow_growing=allow_g, allow_growing_docs=allow_g_docs,
                           want_payload=True)
    if allow_g is not None and allow_g_docs is not None:   # the reference's bitmap: the bits below allow_growing_docs
        bits = np.unpackbits(np.asarray(allow_g, np.uint8), bitorder="little")[:ref_n(ref)]
        bits = np.r_[bits, np.zeros(max(0, ref_n(ref) - len(bits)), np.uint8)]
        bits[allow_g_docs:] = 0
        allow_g = np.packbits(bits, bitorder="little")
    want = ix.search_batch_growing(ref, q_off, q_terms, k, allow=allow, allow_growing=allow_g, want_payload=True)
    return got, want


def ref_n(ref):
    return int(ref.info().n_docs)


def _champion_cut_doc(seg):
    """A document at rank 128 (the last champion) of a term with more than 128 postings in the segment's handle."""
    lay, der = seg.arrays()
    got = read_back(lay, der)
    df = got["df"].astype(np.int64)
    t = int(np.flatnonzero(df > CHAMP_L)[0])
    champ = got["champ"].reshape(-1, 2)
    return int(champ[int(got["champ_off"][t]) + CHAMP_L - 1, 0])


SCRIPT = [("insert", 1), ("insert", 7), ("delete_pending", 3), ("insert", 500), ("delete_indexed", 40),
          ("delete_twice", 2), ("insert", 3000), ("delete_champion", 1), ("insert", 1)]


# (norm form, payload, prune) -> the seed of the script; with seed 20 the first refresh indexes no posting at all (the
# one document of step 0 is deleted on insert): a handle without blocks
SCRIPTS = {("doc_len", False, 1): 1, ("doc_len", True, 0): 20, ("fieldnorm", False, 0): 3, ("fieldnorm", True, 1): 2}


@pytest.mark.parametrize("form,with_payload,prune", list(SCRIPTS))
def test_script_arrays_and_rows(m, orc, world, form, with_payload, prune):
    """After every step of the script and its refresh: every array equals bm25x_growing_create's and the restatement's,
    every search output equals bm25x_search_batch_growing's (k from 1 to 65 535, prefilters on both sides, a growing
    prefilter shorter than the segment), and a subset equals the oracle's restatement of the reference's scan."""
    run_script(orc, world, form, with_payload, prune, SCRIPTS[(form, with_payload, prune)])


def run_script(orc, w, form, with_payload, prune, seed):
    ix, sealed = w["ix"], w["sealed"]
    ix.set_option("prune", prune)
    rng = np.random.default_rng(seed)
    seg = ix.growing_segment()
    docs = Docs()
    q_off, q_terms = _queries(rng, sealed.n_terms, 20)
    allow = np.packbits(rng.random(sealed.n_docs) < 0.7, bitorder="little")
    indexed = 0
    try:
        for step, (op, n) in enumerate(SCRIPT):
            if op == "insert":
                lo = docs.n
                _new_docs(rng, w, docs, n)
                seg.insert(**_kw(docs, form, with_payload, lo, docs.n, orc=orc))
            else:
                if op == "delete_pending":
                    lo = docs.n
                    _new_docs(rng, w, docs, 10, p_deleted=0)
                    seg.insert(**_kw(docs, form, with_payload, lo, docs.n, orc=orc))
                    victims = rng.choice(np.arange(lo, docs.n), size=n, replace=False)
                elif op == "delete_indexed":
                    victims = rng.choice(indexed, size=n, replace=False)
                elif op == "delete_twice":
                    v = int(rng.choice(np.flatnonzero(np.array(docs.deleted[:indexed]) == 0)))
                    victims = np.array([v, v])
                    seg.delete(victims)
                else:
                    victims = np.array([_champion_cut_doc(seg)])
                seg.delete(victims)
                for v in victims:
                    docs.deleted[int(v)] = 1
            assert seg.info().pending == 1
            seg.refresh()
            indexed = docs.n
            info = seg.info()
            assert info.pending == 0 and info.n_docs == docs.n and info.n_deleted == sum(docs.deleted)
            what = f"{form} payload={with_payload} prune={prune} seed {seed} step {step} {op}"
            ref = _reference(w, docs, form, with_payload, orc)
            try:
                _same_arrays(seg, ref, w, docs, form, with_payload, orc, what)
                assert info.n_postings == ref.info().n_postings
                allow_g = np.packbits(rng.random(docs.n) < 0.6, bitorder="little")
                for k in KS:
                    got, want = _search_both(seg, ix, ref, q_off, q_terms, k)
                    same_rows(got, want, f"{what} k={k}")
                for k in (10, 129):
                    got, want = _search_both(seg, ix, ref, q_off, q_terms, k, allow=allow, allow_g=allow_g)
                    same_rows(got, want, f"{what} k={k} prefiltered")
                    short = max(0, docs.n - 5)
                    got, want = _search_both(seg, ix, ref, q_off, q_terms, k, allow_g=allow_g, allow_g_docs=short)
                    same_rows(got, want, f"{what} k={k} allow_growing_docs={short}")
            finally:
                ref.close()
        # the oracle's restatement of search.rs:83-135 + the sealed scan, on a subset
        a = docs.arrays()
        g = orc.GrowingDocs(a["elem_off"], a["elem_term"], a["elem_tf"], a["doc_len"], a["deleted"])
        res = seg.search_batch(q_off, q_terms, 10)
        for i in range(len(q_off) - 1):
            q = q_terms[q_off[i]:q_off[i + 1]]
            if len(np.unique(q[q < sealed.n_terms])) > 32:
                continue
            ed, es = growing_expect(w["oix"], g, sealed.n_docs, q, 10)
            n = int(res["n"][i])
            assert res["doc"][i, :n].tolist() == ed and res["score64"][i, :n].tolist() == es, f"oracle q{i}"
    finally:
        seg.close()
        ix.set_option("prune", 1)


def test_empty_all_deleted_and_refusals(m, orc, world):
    w = world
    ix, sealed = w["ix"], w["sealed"]
    rng = np.random.default_rng(7)
    q_off, q_terms = _queries(rng, sealed.n_terms, 30)
    alone = ix.search_batch(q_off, q_terms, 50, want_payload=True)
    seg = ix.growing_segment()
    try:
        same_rows(seg.search_batch(q_off, q_terms, 50, want_payload=True), alone, "opened, empty")
        docs = Docs()
        _new_docs(rng, w, docs, 300)
        seg.insert(**_kw(docs, "doc_len", False))
        seg.delete(np.arange(docs.n))
        seg.delete(np.arange(docs.n))                       # again: a no-op
        assert seg.info().n_deleted == docs.n
        same_rows(seg.search_batch(q_off, q_terms, 50, want_payload=True), alone, "every document deleted")
        assert seg.info().n_postings == 0
        # a live segment, then every refusal: the segment and its rows stay as they were
        lo = docs.n
        _new_docs(rng, w, docs, 500, p_deleted=0)
        seg.insert(**_kw(docs, "doc_len", False, lo, docs.n))
        before = seg.search_batch(q_off, q_terms, 50, want_payload=True)
        info0 = tuple(getattr(seg.info(), f) for f, _ in m.GrowingInfo._fields_)

        def refused(fn, code, text):
            with pytest.raises(m.Bm25xError) as e:
                fn()
            assert e.value.code == code and text in str(e.value), str(e.value)
            assert tuple(getattr(seg.info(), f) for f, _ in m.GrowingInfo._fields_) == info0

        off = np.array([0, 2], np.uint64)
        refused(lambda: seg.insert(off, [5, 4], [1, 1], doc_len=[2]), 1,
                "bm25x_growing_create: corrupt documents (term ordinals must be strictly ascending per document, tf != 0)")
        refused(lambda: seg.insert(off, [4, 5], [1, 0], doc_len=[2]), 1, "tf != 0")
        refused(lambda: seg.insert(off, [4, 5], [1, 1 << 24], doc_len=[2]), 4, "term frequency >= 2^24")
        refused(lambda: seg.insert(off, [4, 5], [1, 1], doc_fieldnorm=[2]), 1, "doc_fieldnorm")
        refused(lambda: seg.delete([0, docs.n + 3]), 1, f"ordinal {docs.n + 3} (entry 1)")
        refused(lambda: seg.search_batch(q_off, q_terms, 0), 5, "number of needed rows is set to 0")
        refused(lambda: seg.search_batch(q_off, q_terms, 65536), 4, "k=65536")
        wide = np.arange(65, dtype=np.uint32)
        refused(lambda: seg.search_batch(np.array([0, 65], np.uint32), wide, 10), 4, "65 live terms")
        same_rows(seg.search_batch(q_off, q_terms, 50, want_payload=True), before, "after the refusals")
        # the same refusals as bm25x_growing_create's, codes and messages
        for terms, tfs in (([5, 4], [1, 1]), ([4, 5], [1, 1 << 24])):
            with pytest.raises(m.Bm25xError) as a:
                ix.growing(off, terms, tfs, doc_len=[2])
            with pytest.raises(m.Bm25xError) as b:
                seg.insert(off, terms, tfs, doc_len=[2])
            assert (a.value.code, str(a.value)) == (b.value.code, str(b.value))
    finally:
        seg.close()


def test_stats_are_the_sums_plus_the_merge(m, orc, world):
    w = world
    ix, sealed = w["ix"], w["sealed"]
    rng = np.random.default_rng(11)
    docs = Docs()
    _new_docs(rng, w, docs, 2000)
    seg = ix.growing_segment()
    ref = _reference(w, docs, "doc_len", False, orc)
    try:
        seg.insert(**_kw(docs, "doc_len", False))
        q_off, q_terms = _queries(rng, sealed.n_terms, 200)
        seg.refresh()
        for k in (10, 1000):
            st = seg.search_batch(q_off, q_terms, k)["stats"]
            a = ix.search_batch(q_off, q_terms, k)["stats"]
            b = ref.search_batch(q_off, q_terms, k)["stats"]
            for f in ("queries", "postings", "postings_fetched"):
                assert getattr(st, f) == getattr(a, f) + getattr(b, f), (k, f)
            assert st.launches == a.launches + b.launches + 1, k
            old = ix.search_batch_growing(ref, q_off, q_terms, k)["stats"]
            assert old.queries == a.queries and old.launches == st.launches and old.postings == st.postings
    finally:
        ref.close()
        seg.close()


def test_concurrent_searches_see_whole_states(m, orc, world):
    """One thread inserts and deletes through a fixed script; four threads search meanwhile.  Every search returns the
    rows of one state of the script (computed beforehand on bm25x_growing_create handles)."""
    w = world
    ix, sealed = w["ix"], w["sealed"]
    rng = np.random.default_rng(23)
    q_off, q_terms = _queries(rng, sealed.n_terms, 40)
    docs = Docs()
    ops = []
    for i in range(8):
        lo = docs.n
        _new_docs(rng, w, docs, int(rng.integers(1, 300)))
        ops.append(("insert", lo, docs.n))
        if i % 2 and docs.n:
            ops.append(("delete", rng.choice(docs.n, size=min(20, docs.n), replace=False)))
    # the states: after each op, the documents so far with the deletions so far
    states, deleted = [], np.zeros(docs.n, np.uint8)
    empty = ix.search_batch_growing(None, q_off, q_terms, 20, want_payload=True)
    expect = [empty]
    n_now = 0
    for op in ops:
        if op[0] == "insert":
            n_now = op[2]
            deleted[op[1]:op[2]] = docs.deleted[op[1]:op[2]]
        else:
            deleted[op[1]] = 1
        sub = Docs()
        for d in range(n_now):
            e0, e1 = docs.off[d], docs.off[d + 1]
            sub.add(docs.term[e0:e1], docs.tf[e0:e1], deleted[d], docs.payload[d])
        ref = _reference(w, sub, "doc_len", False, orc)
        expect.append(ix.search_batch_growing(ref, q_off, q_terms, 20, want_payload=True))
        ref.close()
    seg = ix.growing_segment()
    errors, seen = [], set()
    stop = threading.Event()
    started, returned = [0], [0]  # ops the writer has begun / that have returned: state i follows op i - 1

    def writer():
        try:
            for i, op in enumerate(ops):
                started[0] = i + 1
                if op[0] == "insert":
                    seg.insert(**_kw(docs, "doc_len", False, op[1], op[2]))
                else:
                    seg.delete(op[1])
                returned[0] = i + 1
        except Exception as e:  # reported by the main thread
            errors.append(e)
        finally:
            stop.set()

    def reader():
        try:
            while True:
                done = stop.is_set()
                lo = returned[0]
                got = seg.search_batch(q_off, q_terms, 20, want_payload=True)
                hi = started[0]
                match = [i for i, e in enumerate(expect) if all(np.array_equal(got[x], e[x]) for x in
                                                                 ("doc", "score", "score64", "payload", "n"))]
                assert match, "a search returned rows of no state of the script"
                # every op that returned before the search began is in it, and no op begun after it ended
                assert any(lo <= i <= hi for i in match), (lo, hi, match)
                seen.add(match[-1])
                if done:
                    break
        except Exception as e:
            errors.append(e)

    threads = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(4)]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors[0]
        assert len(expect) - 1 in seen      # the readers that started after the last op saw the final state
    finally:
        seg.close()


def test_refreshes_free_their_memory(m, orc, world):
    w = world
    ix = w["ix"]
    rng = np.random.default_rng(31)
    docs = Docs()
    _new_docs(rng, w, docs, 400)

    def run(n_refresh):
        seg = ix.growing_segment()
        step = max(1, docs.n // n_refresh)
        for i in range(n_refresh):
            lo, hi = min(i * step, docs.n - 1), min((i + 1) * step, docs.n) if i < n_refresh - 1 else docs.n
            if hi > lo:
                seg.insert(**_kw(docs, "doc_len", False, lo, hi))
            if i % 3 == 2:
                seg.delete([int(rng.integers(hi))])
            seg.refresh()
        seg.close()

    run(3)  # loads every kernel of a refresh before the measurement
    free = free_bytes()
    run(50)
    assert free_bytes() == free, "device memory of the segment not freed"
