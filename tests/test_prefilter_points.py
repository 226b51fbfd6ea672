"""CPU: the prefilter fixtures of test_gpu_prefilter_points.py reach the decisions they were built for (tests/util_prefilter.py).

  champions   every filtered-champion bitmap leaves a top k that needs a document beyond its term's seeds: a seeded
              launch of that batch would miss it.
  two-phase   the hand-over happens before the decisive documents (region L, every other one cleared), after them, or
              never (the pool short of k, or no threshold above a single posting), with pruning on and off.
  pools       the bitmaps allow exactly the matches they name, and the last-window case allows matches of the last
              window only.
  pruning     with the band allowed the head is pruned at the second boundary; with the band cleared no threshold the
              allowed documents give prunes it.
  margin      B meets the allowed k-th A a few ulps away; in the two-phase case, with pruning off, the hand-over comes
              before B (with pruning on the query never suspends).
  dense       the cleared best documents lie in a window the plain kernel sums in its dense accumulator.
  growing     the decisive growing documents are partly cleared and partly past allow_growing_docs, and would be rows
              without the bitmap."""
import numpy as np
import pytest

import util_filter as uf
import util_prefilter as upf
import util_prune as up
from util_segment import growing_expect

_CACHE = {}


def _cached(key, make):
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


def test_bitmap_bits():
    """Bit d of byte d >> 3, least significant first; padding bits only on request."""
    b = upf.bitmap(13, allowed=[0, 9, 12])
    assert b.tolist() == [0b00000001, 0b00010010]
    assert upf.bitmap(13, pad=True).tolist() == [0xFF, 0xFF] and upf.bitmap(13).tolist() == [0xFF, 0x1F]
    assert upf.bitmap(13, cleared=[3]).tolist() == [0xF7, 0x1F]
    assert np.flatnonzero(upf.allowed_mask(b, 13)).tolist() == [0, 9, 12]


def _champions(orc):
    return _cached("champions", lambda: upf.champion_case(orc))


@pytest.mark.parametrize("kind", upf.CHAMP_KINDS)
def test_filtered_champions(orc, kind):
    """Every query, every limit the seeded launch serves (k <= 128): the filtered top k is full and holds a single-term
    document that is not among its term's seeds (at k = 1, all_but_last clears nothing: that limit is left out)."""
    c = _champions(orc)
    assert c.n_docs % 8 != 0
    for k in upf.CHAMP_KS:
        allow = upf.champion_bitmap(c, kind, k)
        for q in c.qs:
            docs, _ = upf.topk(c, q, k, allow)
            assert len(docs) == k
            if k <= 128 and not (kind == "all_but_last" and k == 1):
                assert upf.beyond_seeds(c, q, k, allow), (kind, k, q)
            # without the bitmap the answer is the lead term's seeds
            assert not upf.beyond_seeds(c, q, min(k, 128), None)


def _two_phase(orc):
    return _cached("two", lambda: upf.two_phase_case(orc))


@pytest.mark.parametrize("kind", upf.TWO_KINDS)
def test_two_phase_handover(orc, kind):
    """The suspend test over the chunk boundaries, at every limit, pruning on and off.  before: it must pass at a
    boundary before region L, whose first document is cleared (so the resume launch meets every cleared L document);
    after: it cannot pass before L's first k documents (the top k) are consumed, and must pass
    after them; short / low: it can never pass."""
    c = _two_phase(orc)
    for k in upf.TWO_KS:
        if kind == "short" and k == 1:
            continue
        allow = upf.two_phase_bitmap(c, kind, k)
        for q in c.qs:
            for prune in (1, 0):
                can, must, win = upf.handover(c, q, k, allow, prune)
                what = (kind, k, len(q), prune, can, must)
                if kind == "before":
                    assert must is not None and win[must - 1][1] <= c.L[0], what
                    assert can is not None and win[can - 1][1] > c.E[k - 1], what  # not before k region documents
                elif kind == "after":  # the top k (L's first k: equal scores, doc asc) are in the pool by then
                    assert can is not None and must is not None and win[can - 1][1] > c.L[k - 1], what
                else:
                    assert can is None, what
                top, _ = upf.topk(c, q, k, allow)
                if kind == "before":  # cleared L documents would be rows; allowed ones are, after the hand-over
                    assert set(upf.topk(c, q, k)[0].tolist()) & set(c.L[0::2].tolist())
                    assert set(top.tolist()) & set(c.L[1::2].tolist())
                    assert not set(top.tolist()) & set(c.L[0::2].tolist())
                if kind == "after":
                    assert set(top.tolist()) <= set(c.L.tolist())
                if kind == "short":
                    assert len(top) == k - 1


def _pools(orc):
    return _cached("pools", lambda: upf.pool_case(orc))


def test_unfilled_pool_bitmaps(orc):
    """Each bitmap allows exactly the matches it names (0, 1, k - 1, k, k + 1); the largest limit is served by the HBM
    pool; the last-window bitmaps allow k + 1 matches, all in the last window of the plain kernel."""
    c = _pools(orc)
    assert uf.pool_capacity(65535) > 2048 and uf.pool_capacity(1025) > 2048
    for q in c.qs:
        assert len(upf.matches(c, q)) >= 65536
        for k in (10, 1025):
            for n in (0, 1, k - 1, k, k + 1):
                allow = upf.pool_bitmap(c, q, k, n)
                assert len(upf.topk(c, q, 70000, allow)[0]) == n
    q = c.qs[0]
    for k in upf.LAST_KS:
        allow = upf.last_window_bitmap(c, q, k)
        top, _ = upf.topk(c, q, 70000, allow)
        assert len(top) == k + 1 and top.min() >= upf.last_window(c, q) > 90000


def _prune(orc, name):
    return _cached(("prune", name), lambda: upf.prune_fixture(orc, name))


@pytest.mark.parametrize("name", list(upf.PRUNE_ROLES))
def test_prune_under_bitmap(orc, name):
    """band: the first window holds allowed band documents only and enough of them to cut the pool; at both ends of
    their band the prune set is the head alone.  cleared: the k-th allowed score leaves every term's bound above half of
    it, so nothing can be pruned at any boundary (the pool holds allowed documents only)."""
    c = _prune(orc, name)
    bms = upf.prune_bitmaps(c, upf.PRUNE_KP)
    P, _ = upf.prune_band(c, upf.PRUNE_K, upf.PRUNE_KP, bms["band"])
    assert P == [c.head], (P, c.head)
    P0, _ = upf.prune_band(c, upf.PRUNE_K, upf.PRUNE_KP, upf.bitmap(c.n_docs))
    assert P0 == P
    P, final = upf.prune_band(c, upf.PRUNE_K, upf.PRUNE_KP, bms["cleared"])
    assert P is None and final == []
    assert len(upf.topk(c, c.q, upf.PRUNE_K, bms["cleared"])[0]) == upf.PRUNE_K
    assert up.prune_at(c, [int(t) for t in c.q], float(upf.topk(c, c.q, upf.PRUNE_K, bms["band"])[1][-1]))


@pytest.mark.parametrize("name", list(upf.MARGIN))
def test_margin_under_bitmap(orc, name):
    """With the high documents cleared the filtered top 2 is (B, A); at k = 1 the pool is cut with A in it before B
    (enough allowed documents between them), so B meets Sk = S_A: its f32 filter score is below f32_rd(S_A) (a kernel
    without the margin drops it) and the shipped margin keeps it, with and without the terms pruned at S_A."""
    c = _cached(("margin", name), lambda: upf.margin_case(orc, name))
    allow = upf.margin_bitmap(c)
    oix = orc.OracleIndex(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"],
                                     k1=2.0, b=0.0))
    od, os_, _ = oix.search_exhaustive(c["query"], 2, allow=allow)
    assert od.tolist() == [c["b_doc"], c["a_doc"]] and os_[1] == c["S_a"]
    assert c["tight"] and c["keeps"] and c["tight_pruned"] and c["keeps_pruned"]
    ok = upf.allowed_mask(allow, c["n_docs"])
    between = np.unique(c["post_doc"][(c["post_doc"] > c["a_doc"]) & (c["post_doc"] < c["b_doc"])])
    assert ok[between].sum() >= uf.cut_trigger(1, uf.pool_capacity(1), False)
    if upf.MARGIN[name][1] == "twophase":
        # pruning off: the hand-over comes before B, so the resume launch scores it; pruning on: term x is pruned at
        # S_A and its bound lowers Flo below the streamed terms' bounds, so the suspend launch keeps the query to B
        hi = upf.handover_before(c, 1, allow, 0, c["a_doc"] + 40)
        assert hi is not None and hi <= c["b_doc"], hi
        assert c["pruned"] and upf.handover_before(c, 1, allow, 1, c["a_doc"] + 40) is None


def test_dense_window(orc):
    """The best documents lie in one window that the plain kernel clamps to its accumulator and sums densely; without
    the bitmap they are the top rows, with them cleared the next ones are."""
    c = _cached("dense", lambda: upf.dense_case(orc))
    lo, hi, dense = upf.dense_window(c, c.best)
    assert dense and hi - lo == upf.DENSE_ACC, (lo, hi, dense)
    assert upf.dense_window(c, c.next)[2]
    allow = upf.bitmap(c.n_docs, cleared=c.best)
    for k in upf.DENSE_KS:
        top, _ = upf.topk(c, c.q, k)
        assert set(top.tolist()) & set(c.best)
        top, _ = upf.topk(c, c.q, k, allow)
        assert top[:upf.DENSE_BEST].tolist() == c.next[:k]


def test_growing_bitmap(orc):
    """Sealed two-phase corpus plus growing documents: the rows of every query mix sealed and growing documents; the
    cleared decisive growing documents and those past allow_growing_docs would be rows without the bitmap."""
    c = _two_phase(orc)
    off, term, tf, doc_len, dec = upf.growing_docs(c)
    g = orc.GrowingDocs(off, term, tf, doc_len)
    oix = orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=up.K1, b=up.B))
    ag, cut = upf.growing_bitmap(dec)
    ref = upf.growing_reference_bitmap(ag, cut)
    assert upf.allowed_mask(ag, upf.GROW_N)[cut:].all() and (dec >= cut).any()
    lost = set((c.n_docs + dec[dec < cut][0::2]).tolist()) | set((c.n_docs + dec[dec >= cut]).tolist())
    for k in upf.GROW_KS:
        for q in c.qs:
            q = np.array(q, np.uint32)
            d, _ = growing_expect(oix, g, c.n_docs, q, k, allow=upf.two_phase_bitmap(c, "before", k), allow_g=ref)
            assert any(x >= c.n_docs for x in d) and not set(d) & lost
            d0, _ = growing_expect(oix, g, c.n_docs, q, k)
            assert set(d0) & lost
