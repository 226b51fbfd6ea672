"""GPU: growing segment (SURVEY §8 f3) — bm25::search over sealed + not-yet-sealed documents (search.rs:83-135).

The growing documents are inverted into a second index handle that scores with the sealed segment's statistics
(bm25x_growing_create); a query is two top-k searches and a merge (bm25x_search_batch_growing).  Bar: ids bit-exact
under the canonical rule (score desc, sealed before growing, ascending id), f64 scores bit-exact against the oracle's
restatement of the reference's scan, f32 scores = (float) f64 scores.  (File name: runs after the other GPU tests.)"""
import numpy as np
import pytest

import _pkg
from test_gpu_parity import _oracle_index

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


def _setup(m, orc, seed, n_sealed, n_growing, vocab, extra_vocab, zipf):
    sealed = m.synth_corpus(seed, n_sealed, vocab, 8, 80, zipf)
    fresh = orc.Corpus.synth(seed + 1, n_growing, vocab + extra_vocab, 1, 120, zipf_s=zipf)
    deleted = (np.arange(n_growing) % 5 == 2).astype(np.uint8)
    g = orc.GrowingDocs.from_corpus(fresh, deleted)
    g.elem_term = np.where(g.elem_term >= vocab, m.TERM_MISSING, g.elem_term).astype(np.uint32)
    ix = m.Index.from_corpus(sealed)
    gix = ix.growing(g.elem_off, g.elem_term, g.elem_tf, doc_len=g.doc_len, deleted=deleted)
    return sealed, g, ix, gix, _oracle_index(orc, sealed)


def _expect(oix, g, N, q, k, allow=None, allow_g=None):
    sd, ss, _ = oix.search_exhaustive(q, k, allow=allow)
    gd, gs = oix.search_growing(g, q, k, allow=allow_g)
    rows = sorted([(-s, int(d)) for d, s in zip(sd, ss)] + [(-s, int(d) + N) for d, s in zip(gd, gs)])[:k]
    return [d for _, d in rows], [-s for s, _ in rows]


@pytest.mark.parametrize("cfg", [dict(seed=61, ns=20000, ng=1500, vocab=3000, extra=200, zipf=0.8),
                                 dict(seed=63, ns=3000, ng=3000, vocab=60, extra=5, zipf=1.0)], ids=["sparse", "dense"])
def test_growing_matches_oracle(m, orc, cfg):
    sealed, g, ix, gix, oix = _setup(m, orc, cfg["seed"], cfg["ns"], cfg["ng"], cfg["vocab"], cfg["extra"], cfg["zipf"])
    N = sealed.n_docs
    q_off, q_terms = m.synth_queries(cfg["seed"] + 1000, 60, cfg["vocab"], 1, 8, sealed.post_off, cfg["zipf"])
    for k in (1, 10, 100):
        alone = gix.search_batch(q_off, q_terms, k)
        both = ix.search_batch_growing(gix, q_off, q_terms, k, want_payload=True)
        for i in range(len(q_off) - 1):
            q = q_terms[q_off[i]:q_off[i + 1]]
            gd, gs = oix.search_growing(g, q, k)                     # the growing handle alone
            n = int(alone["n"][i])
            assert n == len(gd) and np.array_equal(alone["doc"][i, :n], gd), f"q{i} k{k} growing ids"
            assert np.array_equal(alone["score64"][i, :n], gs), f"q{i} k{k} growing f64 scores"
            ed, es = _expect(oix, g, N, q, k)                        # sealed + growing, merged
            n = int(both["n"][i])
            assert n == len(ed) and both["doc"][i, :n].tolist() == ed, f"q{i} k{k} merged ids"
            assert both["score64"][i, :n].tolist() == es
            assert np.array_equal(both["score"][i, :n], np.array(es).astype(np.float32)), f"q{i} k{k} merged f32 scores"
            for r in range(n):                                       # default payload = ctid of the segment-local id
                d = int(both["doc"][i, r]) - (N if both["doc"][i, r] >= N else 0)
                assert tuple(both["payload"][i, r]) == ((d // 291) >> 16, (d // 291) & 0xFFFF, d % 291 + 1)
    # no growing handle = the sealed search
    a, b = ix.search_batch_growing(None, q_off, q_terms, 10), ix.search_batch(q_off, q_terms, 10)
    assert np.array_equal(a["doc"], b["doc"]) and np.array_equal(a["score64"], b["score64"])
    gix.close()
    ix.close()


def test_growing_prefilter_and_edges(m, orc):
    sealed, g, ix, gix, oix = _setup(m, orc, 71, 5000, 800, 500, 50, 0.5)
    N = sealed.n_docs
    allow = np.packbits(np.arange(N) % 3 != 0, bitorder="little")
    allow_g = np.packbits(np.arange(g.n_docs) % 2 == 0, bitorder="little")
    qs = [[1, 7, 9], [], [100000], [3], [2, 2, 5, m.TERM_MISSING]]
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    q_terms = np.array([t for q in qs for t in q], dtype=np.uint32)
    res = ix.search_batch_growing(gix, q_off, q_terms, 20, allow=allow, allow_growing=allow_g)
    for i, q in enumerate(qs):
        ed, es = _expect(oix, g, N, np.array(q, dtype=np.uint32), 20, allow=allow, allow_g=allow_g)
        n = int(res["n"][i])
        assert res["doc"][i, :n].tolist() == ed and res["score64"][i, :n].tolist() == es
    assert res["n"][1] == 0 and res["n"][2] == 0
    with pytest.raises(m.Bm25xError, match="number of needed rows is set to 0"):
        ix.search_batch_growing(gix, q_off, q_terms, 0)
    gix.close()
    # a growing segment none of whose tokens the sealed segment knows: every query returns the sealed rows only
    off = np.array([0, 2, 3], dtype=np.uint64)
    lonely = ix.growing(off, [m.TERM_MISSING, m.TERM_MISSING, m.TERM_MISSING], [1, 2, 3], doc_len=[3, 3])
    a, b = ix.search_batch_growing(lonely, q_off, q_terms, 5), ix.search_batch(q_off, q_terms, 5)
    assert np.array_equal(a["doc"], b["doc"]) and np.array_equal(a["n"], b["n"])
    lonely.close()
    # documents must keep the reference's invariants (vector.rs:39-75)
    with pytest.raises(m.Bm25xError, match="strictly ascending"):
        ix.growing(np.array([0, 2], dtype=np.uint64), [5, 4], [1, 1], doc_len=[2])
    with pytest.raises(m.Bm25xError, match="tf != 0"):
        ix.growing(np.array([0, 1], dtype=np.uint64), [5], [0], doc_len=[1])
    ix.close()
