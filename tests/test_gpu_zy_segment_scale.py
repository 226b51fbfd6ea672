"""GPU: the refresh and the seal of a growing segment at the vocabulary size they are built for.  k_splice_count,
k_splice and k_seal_doc_postings take one warp per term in a grid capped at 32 blocks of 8 warps per SM and loop
`t += warps`; with T = 3 x sm_count x 256 terms (101 376 on a 132-SM H100) every warp of every
one of them takes three trips, on whatever card runs this.  Sealed: ~400 k documents of 16-48 terms, Zipf 0.8, the upper
half of the vocabulary thinned to 0-3 postings per term (head lists of ~200 k postings: thousands of 32-posting steps).
Growing: 40 k documents over the same vocabulary, 2000 new ordinals (keyed: new keys that interleave with the sealed
ones) and unknown tokens, in three insert batches with refreshes and deletes in between; 10 % of the sealed and 5 % of
the growing documents are deleted at the seal.

Bit for bit: after each refresh every array of the segment's handle against bm25x_growing_create over the same documents
and the CPU restatement; after the seal every array, pdoc, the champion lists, s1f_min, the info and the three maps against
bm25x_index_create over util_maintain's corpus and util_index.restate over the WHOLE corpus (no sub-vocabulary: it takes
~7 s); bm25x_index_get_df against the restated df; 2000 mixed 1-8-term queries at k = 10, 128, 1025 through the segment
against bm25x_search_batch_growing on the re-created handle, and on the result against the index built from the restated
corpus, 50 of them against the oracle; device memory after the second case equal to that after the first.
Measured on one H100 80GB HBM3 (700 W power limit): ~25 s per case, 53 s for the file, host peak 2.0 GB."""

import numpy as np
import pytest

from util_cuda import free_bytes, sm_count
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_maintain import MISSING, maintain
from util_parity import compare, same_rows
from util_segment import World, check_result, check_segment, docs_from_postings, first_docs, pack, random_keys

pytestmark = pytest.mark.gpu

N_SEALED, N_GROWING, N_NEW = 400_000, 40_000, 2000
KS = (10, 128, 1025)
ROWS = ("doc", "score", "score64", "n")
free_after = {}                                                  # case -> free device bytes once everything is closed


def _sealed(m, rng, T, keyed):
    c = m.synth_corpus(0x5CA1E, N_SEALED, T, 16, 48, 0.8)
    off = c.post_off.astype(np.int64)
    term = np.repeat(np.arange(T), np.diff(off))
    keep = (term < T // 2) | (rng.random(len(term)) < 0.06)      # the tail: 0-3 postings per term
    new_off = np.concatenate([[0], np.cumsum(np.bincount(term[keep], minlength=T))]).astype(np.uint64)
    keys = np.array(sorted(random_keys(np.random.default_rng(T), T).tolist()), np.uint8) if keyed else None
    w = World(m, c.n_docs, new_off, c.post_doc[keep], c.post_tf[keep], c.doc_len.copy(), None, keys)
    c.free()
    return w


def _growing(m, orc, rng, T):
    """Documents over the sealed vocabulary, the ordinals T .. T + N_NEW - 1 and, beyond them, unknown tokens."""
    c = m.synth_corpus(0x5CA1F, N_GROWING, T + N_NEW + 500, 16, 48, 0.8)
    term = np.repeat(np.arange(c.n_terms), np.diff(c.post_off.astype(np.int64)))
    term = np.where(term >= T + N_NEW, MISSING, term)
    docs = docs_from_postings(rng, c.n_docs, term, c.post_doc.astype(np.int64), c.post_tf.copy())
    c.free()
    return docs


@pytest.mark.parametrize("kind", ["keyless", "keyed"])
def test_more_terms_than_warps(m, orc, kind):
    sms = sm_count()
    T = 3 * sms * 256
    assert T >= 3 * (sms * 32) * 8, "the term loops of the refresh and seal kernels take fewer than three trips"
    rng = np.random.default_rng(0x5CA1E)
    keyed = kind == "keyed"
    w = _sealed(m, rng, T, keyed)
    assert w.df.max() > 100_000 and np.count_nonzero(w.df == 0) > 1000 and np.count_nonzero(w.df <= 3) > 10_000
    docs = _growing(m, orc, rng, T)
    new_keys = random_keys(np.random.default_rng(N_NEW), N_NEW, w.keys) if keyed else None   # both cases: the same documents
    q_off, q_terms = m.synth_queries(0x5CA20, 2000, T, 1, 8, w.off, 0.8)
    seg = w.ix.growing_segment()
    got = ref = None
    try:
        lo = 0
        for step, hi in enumerate((20_000, 32_000, N_GROWING)):
            what = f"{kind}, refresh {step}"
            seg.insert(**docs.kw(orc, "doc_len", True, lo, hi))
            if step < 2:
                seg.refresh()
            else:   # the last batch is pending: the searches refresh
                g = w.ix.growing(**docs.kw(orc, "doc_len", True))
                try:
                    for k in KS:
                        same_rows(seg.search_batch(q_off, q_terms, k), w.ix.search_batch_growing(g, q_off, q_terms, k),
                                   f"{kind}, segment k={k}")
                finally:
                    g.close()
            check_segment(orc, seg, w, first_docs(docs, hi), "doc_len", True, what)
            victims = rng.choice(hi, size=int(0.05 * (hi - lo)), replace=False)   # old and new documents alike
            seg.delete(victims)
            docs.deleted[victims] = 1
            lo = hi
        sdel = rng.random(w.n_docs) < 0.1
        got = seg.seal(sealed_deleted=pack(sdel), new_keys=new_keys)
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, "doc_len", True), sealed_deleted=sdel,
                     sealed_keys=w.keys, new_keys=new_keys)
        assert r.n_terms >= 3 * sms * 256, "k_splice's term loop takes fewer than three trips"
        rs = check_result(m, orc, got[0], got[1:], r, f"{kind}, seal")
        assert np.array_equal(got[0].df(), rs.df), f"{kind}: bm25x_index_get_df of the seal's result"
        ref = m.Index(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf, payload=r.payload,
                      term_keys=r.term_keys)
        # the queries in the result's ordinals (keyless: the same), without the terms that vanished
        q_new = r.term_map[q_terms]
        owner = np.repeat(np.arange(len(q_off) - 1), np.diff(q_off.astype(np.int64)))[q_new != MISSING]
        q_new = q_new[q_new != MISSING]
        by_query = np.lexsort((q_new, owner))
        q_new = q_new[by_query].astype(np.uint32)
        q_off = np.concatenate([[0], np.cumsum(np.bincount(owner, minlength=len(q_off) - 1))]).astype(np.uint32)
        oix = orc.OracleIndex(orc.Corpus(r.n_docs, r.doc_len, r.n_terms, r.post_off, r.post_doc, r.post_tf))
        for k in KS:
            rows = got[0].search_batch(q_off, q_new, k)
            same_rows(rows, ref.search_batch(q_off, q_new, k), f"{kind}, result k={k}")
            first = {key: rows[key][:50] for key in ROWS}
            compare(first, oix, q_off[:51], q_new, k, what=f"{kind}, result against the oracle k={k}")
    finally:
        seg.close()
        for ix in (got[0] if got else None, ref, w.ix):
            if ix is not None:
                ix.close()
    free_after[kind] = free_bytes()


def test_device_memory_back_to_baseline():
    """Both cases run the same kernels on corpora of the same shape: once each has closed its handles, the device holds
    what it held after the other."""
    if len(free_after) < 2:
        pytest.skip("needs both cases of test_more_terms_than_warps in this run")
    assert free_after["keyed"] == free_after["keyless"], "device memory of a refresh or a seal not freed"
