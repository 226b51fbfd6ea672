"""CPU: the sparse exact reference of tests/util_sparse.py, which the high-id GPU tests trust, pinned against the oracle's
exhaustive search and util_index.restate on corpora small enough for both; and the high-id corpus checked to hold what it
is built for."""
import numpy as np
import pytest

from util_index import assert_matches, fieldnorms, restate
from util_sparse import DOC_INF, MAX_N_DOCS, T31, SparseReference, high_id_corpus, reference, sum_len_of

KB = [(1.2, 0.75), (2.0, 0.0), (1.2, 1.0)]


@pytest.mark.parametrize("k1,b", KB, ids=[f"k1={a}_b={b}" for a, b in KB])
def test_sparse_reference_equals_oracle_and_restatement(orc, k1, b):
    c = orc.Corpus.synth_bulk(0x5A85E + int(10 * k1 + b * 4), 60000, 800, 1, 90, 0.8, k1=k1, b=b)
    fn = fieldnorms(orc, c.doc_len)
    sum_len = int(c.doc_len.astype(np.uint64).sum())
    ref = SparseReference(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, k1, b, sum_len, fieldnorm=fn)
    oix = orc.OracleIndex(c)
    rng = np.random.default_rng(3)
    allow = np.packbits(rng.random(c.n_docs) < 0.4, bitorder="little")
    df = np.diff(c.post_off.astype(np.int64))
    queries = [rng.choice(c.n_terms, int(n), replace=False) for n in (1, 1, 2, 3, 5, 8, 17, 40)]
    queries += [[0, 0, 5], [int(np.argmax(df))], [c.n_terms + 3, 7], []]   # duplicates, the longest list, unknown ids
    for q in queries:
        for k in (1, 10, 1000):
            for al in (None, allow):
                od, os_, _ = oix.search_exhaustive(np.asarray(q, np.uint32), k, allow=al)
                got = ref.search(q, k, allow=al)
                assert got.n == len(od) and np.array_equal(got.doc, od), (q, k)
                assert np.array_equal(got.score64, os_), (q, k)
                assert np.array_equal(got.score, os_.astype(np.float32))
    r = restate(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, k1, b, doc_len=c.doc_len)
    a = ref.arrays()

    class Lay:  # restate's scalars in the shape assert_matches reads from a handle
        pass

    lay, der = Lay(), Lay()
    for name in ("n_docs", "n_terms", "n_postings", "n_postings_padded", "n_blocks", "sum_doc_len", "k1", "b", "avgdl"):
        setattr(lay, name, getattr(a, name))
    der.n_champ, der.s1f_min = a.n_champ, a.s1f_min
    got = {name: getattr(a, name) for name in ("post", "post_off", "df", "blk_off", "blk", "s0f", "s0d", "s1d", "s1f",
                                               "ubd", "blk_ub", "pdoc", "champ", "champ_off")}
    assert_matches(got, lay, der, r, f"sparse k1={k1} b={b}", skip=("fieldnorm", "payload"))


def test_high_id_corpus_holds_its_cases(orc):
    """What the GPU tests rely on the corpus for, checked without a GPU (and without its 4 GB of per-document arrays)."""
    N = MAX_N_DOCS - 64
    c = high_id_corpus(N)
    live = c.live
    assert live[0] == 0 and live[-1] == N - 1 and {T31 - 1, T31, T31 + 1} <= set(live.tolist())
    assert np.any((live >= 3 << 30) & (live < (3 << 30) + (1 << 20)))
    off = c.post_off.astype(np.int64)
    lst = lambda t: c.post_doc[off[t]:off[t + 1]].astype(np.int64)
    # pad slots after the largest id
    (p,) = c.kinds["pad"]
    assert lst(p)[-1] == N - 1 and len(lst(p)) % 4 != 0
    # blocks of head terms across 2^31
    straddle = 0
    for t in c.kinds["head"]:
        d = lst(t)
        first, last = d[::128], d[np.minimum(np.arange(0, len(d), 128) + 127, len(d) - 1)]
        straddle += int(np.sum((first < T31) & (last >= T31)))
    assert straddle >= 1
    # the wide term's blocks: bit width 32, then byte width 4
    (w,) = c.kinds["wide"]
    d = lst(w).astype(np.uint32)
    md0, _ = orc.compress_document_ids(int(d[0]), d[:128])
    md1, pd1 = orc.compress_document_ids(int(d[128]), d[128:])
    assert md0 == 32 and md1 == 0x80 | 4 and d[128] >= T31 and np.diff(d[128:].astype(np.int64)).max() >= 1 << 24
    assert np.array_equal(pd1.view("<u4"), d[128:])
    # dense terms: hundreds of postings inside the top 2048 ids
    for t in c.kinds["dense"]:
        assert len(lst(t)) >= 300 and lst(t)[0] >= N - 2048
    # tie groups straddle 2^31 at the champion cut and at limits 128 / 129 / 224 (single-term rows)
    ref = reference(orc, c, 1.2, 0.75)
    for t in c.kinds["tie"]:
        r = ref.search([t], 300)
        ids, s = r.doc.astype(np.int64), r.score64
        for cut in [x for x in (128, 129, 224) if x < r.n]:
            assert s[cut - 1] == s[cut] and ids[cut - 1] >= T31, (t, cut)
        grp = ids[s == s[127]]
        assert grp.min() < T31 <= grp.max()
    # a query matching more than 65 535 documents
    assert ref.search(c.kinds["head"][:3], 65535).n == 65535
    assert sum_len_of(orc, c) > N and DOC_INF == MAX_N_DOCS + 1
