"""Growing segment (SURVEY §8 f3): the oracle's restatement of the scan in bm25::search (search.rs:83-135) against a
pure-Python restatement of the same lines, and the product's host-side merge of two top-k result sets."""
import math

import numpy as np
import pytest

import _pkg


def _py_growing(orc, oix, sealed, g, terms, k):
    """search.rs:49-135 line by line in Python floats (IEEE f64, same operation order)."""
    N = sealed.n_docs
    avgdl = float(int(sealed.doc_len.astype(np.uint64).sum())) / float(N)
    k1, b = 1.2, 0.75
    tokens = sorted({int(t) for t in terms if t < sealed.n_terms and oix.df(int(t)) > 0})   # search.rs:55-62
    out = []
    for d in range(g.n_docs):
        if g.deleted is not None and g.deleted[d]:
            continue
        length = float(orc.lib().orc_fieldnorm_to_length(int(g.fieldnorm[d])))
        result = 0.0
        for e in range(int(g.elem_off[d]), int(g.elem_off[d + 1])):
            t, tf = int(g.elem_term[e]), float(g.elem_tf[e])
            if t in tokens:
                s0 = math.log((float(N) + 1.0) / (float(oix.df(t)) + 0.5)) * (k1 + 1.0)       # bm25.rs:285-289,348
                s1 = k1 * (1.0 - b + b * length / avgdl)                                         # bm25.rs:349-352
                result += (tf * s0) / (tf + s1)                                                  # bm25.rs:355-358
        if 0.0 < result:
            out.append((-result, d))
    out.sort()
    return [d for _, d in out[:k]], [-s for s, _ in out[:k]]


def test_oracle_growing_scan_matches_python_restatement(orc):
    sealed = orc.Corpus.synth(0xB25C0DE0 + 51, 800, 120, 8, 40, zipf_s=0.6)
    fresh = orc.Corpus.synth(0xB25C0DE0 + 52, 150, 140, 1, 60, zipf_s=0.6)      # 20 tokens the sealed segment lacks
    deleted = (np.arange(150) % 7 == 3).astype(np.uint8)
    g = orc.GrowingDocs.from_corpus(fresh, deleted)
    g.elem_term = np.where(g.elem_term >= sealed.n_terms, 0xFFFFFFFF, g.elem_term).astype(np.uint32)
    oix = orc.OracleIndex(sealed)
    rng = np.random.default_rng(7)
    for _ in range(40):
        terms = rng.integers(0, 130, rng.integers(1, 6)).astype(np.uint32)
        for k in (1, 5, 200):
            gd, gs = oix.search_growing(g, terms, k)
            pd_, ps = _py_growing(orc, oix, sealed, g, terms, k)
            assert gd.tolist() == pd_ and gs.tolist() == ps
            assert not any(deleted[d] for d in gd)
    # prefilter bitmap over growing ordinals; empty / unknown-only queries
    allow = np.packbits((np.arange(150) % 2 == 0), bitorder="little")
    gd, _ = oix.search_growing(g, [1, 2, 3], 50, allow=allow)
    assert len(gd) and all(d % 2 == 0 for d in gd)
    assert len(oix.search_growing(g, [5000], 5)[0]) == 0 and len(oix.search_growing(g, [], 5)[0]) == 0


def test_merge_topk_host():
    m = _pkg.load()
    m.build_library()
    rng = np.random.default_rng(11)
    nq, k = 300, 7

    def side(base, ids_below=1000):
        n = rng.integers(0, k + 1, nq).astype(np.uint32)
        doc = np.full((nq, k), 0xFFFFFFFF, np.uint32)
        s64 = np.zeros((nq, k))
        pay = np.zeros((nq, k, 3), np.uint16)
        for q in range(nq):
            sc = np.sort(rng.integers(1, 6, n[q]).astype(np.float64))[::-1] / 4.0    # many equal scores
            ids = np.zeros(n[q], np.uint32)
            for s in np.unique(sc):                                                   # ids ascend inside a tie group
                sel = sc == s
                ids[sel] = np.sort(rng.choice(ids_below, sel.sum(), replace=False))
            doc[q, :n[q]], s64[q, :n[q]] = ids, sc
            pay[q, :n[q], 0] = ids % 65536
            pay[q, :n[q], 2] = base
        return {"doc": doc, "score": s64.astype(np.float32), "score64": s64, "payload": pay, "n": n}

    # list b at the top of the id space: doc_base_b + k - 1 is the largest doc id, 0xFFFFFFFD (0xFFFFFFFF marks empty slots)
    for doc_base_b, b_ids_below in ((5000, 1000), (0xFFFFFFFE - k, k)):
        a, b = side(1), side(2, b_ids_below)
        out = m.merge_topk(a, b, doc_base_b, k)
        for q in range(nq):
            rows = [(-a["score64"][q, i], int(a["doc"][q, i]), 1) for i in range(a["n"][q])] + \
                   [(-b["score64"][q, i], int(b["doc"][q, i]) + doc_base_b, 2) for i in range(b["n"][q])]
            rows.sort()
            rows = rows[:k]
            n = int(out["n"][q])
            assert n == len(rows)
            assert out["doc"][q, :n].tolist() == [r[1] for r in rows]
            assert out["score64"][q, :n].tolist() == [-r[0] for r in rows]
            assert out["payload"][q, :n, 2].tolist() == [r[2] for r in rows]
            assert np.all(out["doc"][q, n:] == 0xFFFFFFFF)
    assert out["doc"].max(initial=0, where=out["doc"] != 0xFFFFFFFF) == 0xFFFFFFFD
    # one id past the largest would come back as the empty-slot marker, two past as document 0: refused
    for over in (k, k + 1):
        q = int(np.flatnonzero(b["n"] > 0)[0])
        bad = {x: v.copy() for x, v in b.items()}
        bad["doc"][q, int(b["n"][q]) - 1] = over
        with pytest.raises(m.Bm25xError, match="exceeds the largest doc id") as e:
            m.merge_topk(a, bad, doc_base_b, k)
        assert e.value.code == 1
    with pytest.raises(m.Bm25xError, match="number of needed rows is set to 0"):
        m.merge_topk({x: (v[:, :0] if v.ndim > 1 else v) for x, v in a.items()},
                     {x: (v[:, :0] if v.ndim > 1 else v) for x, v in b.items()}, 0, 0)
