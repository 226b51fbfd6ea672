"""GPU: the refresh and the seal of a growing segment off the defaults.  One seeded script (insert, refresh, delete,
insert, seal, open a segment on the result, insert, search) runs
- over k1 / b across the range bm25x_index_create accepts, b = 0 and k1 = 0 included, where whole lists tie and the
  champion cut falls by new doc id inside a tie group of sealed and growing documents: the segment's handle against
  bm25x_growing_create and the restatement with the same k1 / b, the seal's result against bm25x_index_create and the
  restatement with them, its searches against the oracle on every kernel path;
- with every kind of finalized handle as the sealed side: ingested from stored blocks with exact lengths, with stored norms
  and the caller's sum of lengths, and a finalized replica of a keyed index (which has no keys: it seals as a keyless one).
Then bm25x_evaluate_batch on a seal's result, whose idf table comes from the host df the seal left."""
from types import SimpleNamespace

import numpy as np
import pytest

from util_cuda import D2D, cudart
from util_index import CHAMP_L, fieldnorms
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_maintain import maintain
from util_parity import live_queries
from util_segment import (Docs, World, check_result, check_searches, check_segment, first_docs, new_docs, pack,
                          random_keys, sealed_docs)

pytestmark = pytest.mark.gpu

KS = (1, 10, 128, 129)
ROWS = ("doc", "score", "score64", "payload", "n")
N, T, N_NEW = 2500, 160, 6
TIE, TIE_TF = 5, 7          # a term with 100 sealed and 60 growing postings of one tf, above every other tf of the corpus


def _corpus(orc, rng, keyed):
    """The sealed documents of util_segment.sealed_docs, 100 of them with the tie term."""
    docs, dead = sealed_docs(rng, N, T)
    for d in range(100, 200):
        docs[d][TIE] = TIE_TF
    c = orc.Corpus.from_docs(docs, n_terms=T)
    return SimpleNamespace(docs=docs, dead=dead, off=c.post_off, doc=c.post_doc, tf=c.post_tf,
                           doc_len=c.doc_len + rng.integers(0, 5, size=N).astype(np.uint32),
                           payload=rng.integers(0, 65536, size=(N, 3)).astype(np.uint16),
                           keys=np.array(sorted(random_keys(rng, T).tolist()), np.uint8) if keyed else None)


def _world(m, c, k1, b, ix=None, keys=None):
    return World(m, N, c.off, c.doc, c.tf, c.doc_len, c.payload, keys, ix, k1, b)


def _script(m, orc, rng, w, c, form, what):
    """The script on the sealed World w (closed at the end, with everything made from it)."""
    k1, b, keyed = w.k1, w.b, w.keys is not None
    new_keys = random_keys(rng, N_NEW, w.keys) if keyed else None
    docs = Docs()
    new_docs(rng, w, c.dead, docs, 100, N_NEW)
    for i in range(60):                                          # the growing part of the tie group
        docs.add([TIE], [TIE_TF], i % 3, False, rng.integers(0, 65536, size=3).tolist())
    copy = sorted(c.docs[7].items())                             # a growing copy of sealed document 7
    docs.add([t for t, _ in copy], [f for _, f in copy], 0, False, [7, 7, 7])
    new_docs(rng, w, c.dead, docs, 50, N_NEW)
    seg = w.ix.growing_segment()
    made = [w.ix]
    try:
        seg.insert(**docs.kw(orc, form, True, 0, 100))
        seg.refresh()
        check_segment(orc, seg, w, first_docs(docs, 100), form, True, f"{what}, first refresh", k1, b)
        victims = rng.choice(100, size=15, replace=False)
        seg.delete(victims)
        for v in victims:
            docs.deleted[int(v)] = 1
        seg.insert(**docs.kw(orc, form, True, 100, docs.n))
        seg.refresh()
        check_segment(orc, seg, w, docs, form, True, f"{what}, second refresh", k1, b)
        sdel = rng.random(N) < 0.1
        sdel[7] = False
        got = seg.seal(sealed_deleted=pack(sdel), new_keys=new_keys)
        made.append(got[0])
        r = maintain(N, w.off, w.doc, w.tf, docs.restated(orc, form, True), sealed_deleted=sdel, sealed_payload=w.payload,
                     sealed_keys=w.keys, new_keys=new_keys)
        # the tie group: more than 128 postings of one tf, fewer than 128 of them sealed
        tie = int(r.term_map[TIE])
        lo, hi = int(r.post_off[tie]), int(r.post_off[tie + 1])
        group = r.post_doc[lo:hi][r.post_tf[lo:hi] == TIE_TF]
        n_sealed = int((~sdel).sum())
        above = int(np.count_nonzero(r.post_tf[lo:hi] > TIE_TF))   # a growing tf of 2^24 - 1 now and then
        assert len(group) > CHAMP_L and 0 < np.count_nonzero(group < n_sealed) < CHAMP_L - above
        rs = check_result(m, orc, got[0], got[1:], r, f"{what}, seal", k1, b)
        if b == 0:   # the score is a function of tf alone: the list ends with the group's first new ids, growing ones last
            champ = rs.champ.reshape(-1, 2)[int(rs.champ_off[tie]):int(rs.champ_off[tie + 1]), 0]
            assert np.array_equal(champ[above:], group[:CHAMP_L - above]) and champ[-1] >= n_sealed
        a, s = got[0].info(), w.ix.info()
        assert (a.k1, a.b) == (s.k1, s.b) == (k1, b), f"{what}: the result's k1 / b"
        check_searches(orc, got[0], r, rng, f"{what}, seal", k1, b, ks=KS)
        # a segment on the result
        w2 = World.from_restated(m, r, got[0], k1, b)
        docs2 = Docs()
        new_docs(rng, w2, np.flatnonzero(w2.df == 0).tolist(), docs2, 80, N_NEW)
        seg2 = w2.ix.growing_segment()
        try:
            seg2.insert(**docs2.kw(orc, form, True))
            g = w2.ix.growing(**docs2.kw(orc, form, True))
            try:
                q_off, q_terms = live_queries(rng, w2.df, [1, 2, 2, 3, 4, 5, 8, 12])
                for k in KS:
                    x = seg2.search_batch(q_off, q_terms, k, want_payload=True)
                    y = w2.ix.search_batch_growing(g, q_off, q_terms, k, want_payload=True)
                    for key in ROWS:
                        assert np.array_equal(x[key], y[key]), f"{what}, segment on the result k={k}: {key}"
            finally:
                g.close()
            check_segment(orc, seg2, w2, docs2, form, True, f"{what}, segment on the result", k1, b)
        finally:
            seg2.close()
        return got, r
    finally:
        seg.close()
        for ix in made:
            ix.close()


K1_B = [(1.2, 0.75), (2.0, 0.0), (0.0, 0.75), (1.2, 1.0), (0.5, 0.3)]


@pytest.mark.parametrize("k1,b", K1_B)
def test_script_over_k1_b(m, orc, k1, b):
    rng = np.random.default_rng(K1_B.index((k1, b)) + 61)
    keyed = k1 != 1.2            # three keyed, two keyless
    c = _corpus(orc, rng, keyed)
    _script(m, orc, rng, _world(m, c, k1, b, keys=c.keys), c, "doc_len" if b else "fieldnorm", f"k1={k1} b={b}")


def _blocks(m, orc, c, k1, b, **kw):
    eb = orc.EncodedBlocks(orc.Corpus(N, c.doc_len, T, c.off, c.doc, c.tf))
    return m.Index.from_blocks(N, T, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf, eb.doc_off, eb.tf_off,
                               eb.bytes[:eb.n_bytes], k1=k1, b=b, payload=c.payload, term_keys=c.keys, **kw)


@pytest.mark.parametrize("kind", ["blocks-doc_len", "blocks-fieldnorm", "replica"])
def test_script_over_handle_kinds(m, orc, kind):
    k1, b = 0.9, 0.4
    rng = np.random.default_rng(71 + len(kind))
    c = _corpus(orc, rng, True)
    if kind == "blocks-doc_len":
        w = _world(m, c, k1, b, _blocks(m, orc, c, k1, b, doc_len=c.doc_len), c.keys)
    elif kind == "blocks-fieldnorm":
        # stored norms hold no exact length: the segment's avgdl comes from the sum the caller gave
        total = int(c.doc_len.astype(np.uint64).sum()) + 777
        w = _world(m, c, k1, b, _blocks(m, orc, c, k1, b, doc_fieldnorm=fieldnorms(orc, c.doc_len), sum_doc_len=total),
                   c.keys)
        w.sum_len = total
    else:
        src = m.Index(N, c.doc_len, T, c.off, c.doc, c.tf, k1=k1, b=b, payload=c.payload, term_keys=c.keys)
        lay = src.layout()
        rep = m.Index.alloc_replica(lay, 0)
        with pytest.raises(m.Bm25xError) as e:
            rep.growing_segment()
        assert e.value.code == 1 and "replica not finalized" in str(e.value)
        rl = rep.layout()
        for i in range(len(rl.dev_ptr)):
            assert cudart().cudaMemcpy(rl.dev_ptr[i], lay.dev_ptr[i], lay.bytes[i], D2D) == 0
        rep.finalize_replica()
        src.close()
        # the keys do not travel with the 13 arrays: the replica answers and seals as a keyless index
        with pytest.raises(m.Bm25xError) as e:
            rep.lookup_terms(c.keys[:3])
        assert e.value.code == 1 and "without term keys" in str(e.value)
        seg = rep.growing_segment()
        try:
            seg.insert([0, 1], [T + 1], [1], doc_len=[1])
            with pytest.raises(m.Bm25xError) as e:
                seg.seal(new_keys=random_keys(rng, 2, c.keys))
            assert e.value.code == 1 and "without term keys" in str(e.value)
        finally:
            seg.close()
        w = _world(m, c, k1, b, rep)
    keyed = w.keys is not None
    (ix, smap, gmap, tmap), r = _script(m, orc, rng, w, c, "doc_len", kind)
    if not keyed:    # stable ordinals, every one of them a term
        assert r.term_keys is None and np.array_equal(tmap, np.arange(len(tmap), dtype=np.uint32)) and len(tmap) == r.n_terms


def test_evaluate_on_a_seals_result(m, orc):
    """bm25x_evaluate_batch builds its idf table from the handle's host df and n_docs: on a seal's result, over unknown
    ordinals, a term whose df the seal brought to 0 and a document whose Σ tf saturates at 2^32 - 1, bitwise against the
    oracle over the restated corpus."""
    rng = np.random.default_rng(83)
    c = _corpus(orc, rng, False)
    w = _world(m, c, 1.2, 0.75)
    docs = Docs()
    new_docs(rng, w, c.dead, docs, 120, N_NEW)
    gone = int(np.flatnonzero((w.df > 0) & (w.df < 40))[0])                 # every document that holds it is deleted
    sdel = np.zeros(N, bool)
    sdel[w.doc[int(w.off[gone]):int(w.off[gone + 1])]] = True
    sdel |= rng.random(N) < 0.05
    seg = w.ix.growing_segment()
    got = None
    try:
        seg.insert(**docs.kw(orc, "doc_len", True))
        victims = [d for d in range(docs.n) if gone in docs.term[docs.off[d]:docs.off[d + 1]]]
        seg.delete(np.array(victims, np.uint32))
        for v in victims:
            docs.deleted[v] = 1
        got = seg.seal(sealed_deleted=pack(sdel))
        r = maintain(N, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", True), sealed_deleted=sdel,
                     sealed_payload=w.payload)
        df = np.diff(r.post_off.astype(np.int64))
        assert df[gone] == 0 and w.df[gone] > 0 and r.n_terms > T
        assert np.array_equal(got[0].df(), df.astype(np.uint32))
        oix = orc.OracleIndex(orc.Corpus(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf))
        pairs_d, pairs_q = [], []
        for i in range(200):
            vocab = r.n_terms + 20                                           # the last 20 ordinals are unknown
            t = set(rng.choice(vocab, size=int(rng.integers(0, 40)), replace=False).tolist())
            q = set(rng.choice(vocab, size=int(rng.integers(0, 9)), replace=False).tolist())
            if i % 4 == 0:
                t.add(gone)
                q.add(gone)
            t, q = np.array(sorted(t), np.uint32), np.array(sorted(q), np.uint32)
            tf = rng.integers(1, 9, size=len(t)).astype(np.uint32)
            if i % 50 == 1:                                                  # Σ tf saturates
                t, tf = np.union1d(t, [1, 2]).astype(np.uint32), None
                tf = np.full(len(t), 0xFFFFFFFF, np.uint32)
                q = np.union1d(q, [1, 2]).astype(np.uint32)
            pairs_d.append(m.Document(t, tf))
            pairs_q.append(m.Query(q))
        assert any(int(d.tfs.astype(np.uint64).sum()) > 0xFFFFFFFF for d in pairs_d)
        have = got[0].evaluate_batch(pairs_d, pairs_q)
        want = np.array([oix.evaluate(d.terms, d.tfs, q.terms) for d, q in zip(pairs_d, pairs_q)])
        assert np.array_equal(have, want) and np.count_nonzero(want) > 40
    finally:
        seg.close()
        if got:
            got[0].close()
        w.ix.close()
