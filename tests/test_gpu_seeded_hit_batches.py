"""GPU: the seeded kernel's hit list.  A seeded launch (RING_SEEDED) does its ring searches per verification pass but
scores the documents they confirm later, several passes and windows at a time (word loads, f32 filter, exact f64 score,
pool insert); the list is flushed when a pass's rows might not fit and once at query end.  These corpora make the list
fill many times per window and across windows (correlated lists: most documents of a query hold two or three of its
terms), put a query's only hits in its last window, flood the k-th score with exact ties, and make seeds that another
run holds.  Every case runs seeded with no hand-back (seed_prune_min / seed_dense_div off) and on the plain kernel:
doc ids, f32 and f64 scores, counts and the unused slots (0xFFFFFFFF) must be the same bits, and equal to the oracle."""
import numpy as np
import pytest

import _pkg
from test_gpu_parity import _compare, _csr_corpus, _PrefixOracle, _rows_identical

pytestmark = pytest.mark.gpu

SEEDED = dict(seed=1, twophase=0, seed_max_terms=8, seed_prune_min=0xFFFFFFFF, seed_dense_div=0)
PLAIN = dict(seed=0, twophase=0)
KS = (1, 10, 64, 128)


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


def _set(ix, **opts):
    for name, value in opts.items():
        ix.set_option(name, value)


def _queries(qs):
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    return q_off, np.array([t for q in qs for t in q], dtype=np.uint32)


def _both_paths(m, ix, oix, qs, what, ks=KS):
    """Seeded and plain launches at every limit: identical rows, equal to the oracle."""
    q_off, q_terms = _queries(qs)
    for k in ks:
        got = {}
        for name, opts in dict(seeded=SEEDED, plain=PLAIN).items():
            for prune in (1, 0):
                _set(ix, prune=prune, **opts)
                got[name, prune] = ix.search_batch(q_off, q_terms, k)
        for key, res in got.items():
            _rows_identical(res, got["plain", 1], f"{what} {key} k={k}")
            assert np.all(res["doc"][np.arange(k)[None, :] >= res["n"][:, None]] == 0xFFFFFFFF), f"{what} {key} k={k}"
        _compare(got["seeded", 0], oix, q_off, q_terms, k, what=f"{what} k={k}")


def _correlated(rng, n_docs, groups, size, share, tf_hi, extra_len):
    """`groups` groups of 8 terms; a group's terms draw most postings from one common pool of `size` documents (a term
    holds each pool document with probability `share`), plus a few of their own: documents hold 2..8 terms of their
    group.  Lists stay far below n_docs / 64."""
    lists = []
    for _ in range(groups):
        pool = rng.choice(n_docs, size=size, replace=False)
        for _ in range(8):
            own = rng.choice(n_docs, size=size // 10, replace=False)
            d = np.unique(np.concatenate([pool[rng.random(size) < share], own]))
            lists.append((d, rng.integers(1, tf_hi + 1, size=len(d))))
    return _csr_corpus(rng, n_docs, lists, extra_len=extra_len)


@pytest.mark.parametrize("share", [0.5, 0.9])
def test_correlated_lists_fill_the_list_often(m, orc, share):
    """Correlated lists over 400k documents: thousands of documents per query hold two or more of its terms, so a
    window lists many hits and the hit list is flushed many times inside one window and across windows.  Every class
    of the seeded kernel (2, 3, 4 and 5..8 terms)."""
    rng = np.random.default_rng(301 + int(share * 10))
    n_docs = 400000
    doc_len, off, pd_, pt = _correlated(rng, n_docs, 6, 4000, share, 6, 40)
    T = len(off) - 1
    assert int(np.diff(off).max()) < n_docs // 64
    ix = m.Index(n_docs, doc_len, T, off, pd_, pt)
    oix = _PrefixOracle(orc.OracleIndex(orc.Corpus(n_docs, doc_len, T, off, pd_, pt)), max(KS))
    qs = []
    for g in range(6):
        base = 8 * g
        for n in (2, 3, 4, 5, 6, 8):
            qs.append(sorted(rng.choice(8, size=n, replace=False) + base))
    qs.append([0, 8, 16])  # terms of different groups: few shared documents, mostly seeds
    _both_paths(m, ix, oix, qs, f"correlated share={share}")
    ix.close()


def test_hits_only_in_the_last_window(m, orc):
    """Term 0 spreads 6000 postings over the whole doc range; terms 1..3 hold documents of the last 3000 ids only, half
    of them shared with term 0 and each other.  Every hit of these queries falls in the last windows, and the rows still
    listed when the stream ends are scored by the flush at query end."""
    rng = np.random.default_rng(311)
    n_docs = 300000
    tail = np.arange(n_docs - 3000, n_docs)
    t0 = np.unique(np.concatenate([rng.choice(n_docs - 3000, size=5000, replace=False), rng.choice(tail, 1000, replace=False)]))
    lists = [(t0, rng.integers(1, 5, size=len(t0)))]
    for _ in range(3):
        d = np.sort(rng.choice(tail, size=1500, replace=False))
        lists.append((d, rng.integers(1, 5, size=len(d))))
    for _ in range(4):  # fillers: varied norms
        d = np.sort(rng.choice(n_docs, size=3000, replace=False))
        lists.append((d, rng.integers(1, 5, size=len(d))))
    doc_len, off, pd_, pt = _csr_corpus(rng, n_docs, lists, extra_len=30)
    T = len(lists)
    ix = m.Index(n_docs, doc_len, T, off, pd_, pt)
    oix = _PrefixOracle(orc.OracleIndex(orc.Corpus(n_docs, doc_len, T, off, pd_, pt)), max(KS))
    qs = [[0, 1], [0, 2, 3], [0, 1, 2, 3], [1, 2, 3], [0, 1, 2, 3, 4, 5], [0, 1, 2, 3, 4, 5, 6, 7]]
    _both_paths(m, ix, oix, qs, "last window")
    ix.close()


@pytest.mark.parametrize("k1", [1.2, 2.0])
def test_tie_flood_across_flushes(m, orc, k1):
    """b = 0 and tf = 1 almost everywhere: a document's score depends only on which terms it holds, so thousands of
    documents tie exactly, and a tie group straddles many flushes of the hit list.  Terms 0..3 are correlated (pairs
    and triples tie among themselves); term 4's postings are held by no other query term (its seeds all enter alone and
    tie with each other and with the k-th entry)."""
    rng = np.random.default_rng(321)
    n_docs = 60000
    pool = rng.choice(40000, size=4000, replace=False)
    lists = []
    for _ in range(4):
        d = np.unique(np.concatenate([pool[rng.random(4000) < 0.6], rng.choice(40000, size=200, replace=False)]))
        tf = np.ones(len(d), np.uint32)
        tf[rng.random(len(d)) < 0.02] = 2
        lists.append((d, tf))
    d4 = np.arange(40000, 42000)
    lists.append((d4, np.ones(len(d4), np.uint32)))
    for _ in range(3):  # fillers: document lengths vary (irrelevant at b = 0, kept for the norms)
        d = np.sort(rng.choice(n_docs, size=5000, replace=False))
        lists.append((d, rng.integers(1, 7, size=len(d))))
    doc_len, off, pd_, pt = _csr_corpus(rng, n_docs, lists, extra_len=200)
    T = len(lists)
    ix = m.Index(n_docs, doc_len, T, off, pd_, pt, k1=k1, b=0.0)
    oix = _PrefixOracle(orc.OracleIndex(orc.Corpus(n_docs, doc_len, T, off, pd_, pt, k1=k1, b=0.0)), max(KS) + 1)
    qs = [[0, 1], [0, 1, 2], [0, 1, 2, 3], [0, 4], [0, 1, 4], [1, 2, 3, 4], [0, 1, 2, 3, 4], [0, 1, 2, 3, 4, 5, 6, 7]]
    _both_paths(m, ix, oix, qs, f"tie flood k1={k1}")
    # the cut falls inside a tie group: the k-th row ties with the (k+1)-th the oracle ranks behind it
    q = np.array(qs[1], np.uint32)
    s = oix.search_exhaustive(q, max(KS) + 1)[1]
    assert any(s[k - 1] == s[k] for k in KS), "no limit cuts a tie group"
    ix.close()


def test_seeds_held_by_another_run(m, orc):
    """Every champion of term 0 (its highest-tf postings) is also held by term 1 or 2, so the seeds of term 0 are all
    the stream's business; term 3's champions are held by nobody else.  No document may appear twice, and the counts
    match the oracle."""
    rng = np.random.default_rng(331)
    n_docs = 200000
    top = np.sort(rng.choice(n_docs, size=300, replace=False))
    rest = np.setdiff1d(rng.choice(n_docs, size=4000, replace=False), top)
    d0 = np.union1d(top, rest)
    tf0 = np.where(np.isin(d0, top), 9, 1).astype(np.uint32)
    half = rng.random(len(top)) < 0.5
    d1 = np.union1d(top[half], rng.choice(n_docs, size=3000, replace=False))
    d2 = np.union1d(top[~half], rng.choice(n_docs, size=3000, replace=False))
    d3 = np.setdiff1d(rng.choice(n_docs, size=3000, replace=False), np.concatenate([d0, d1, d2]))
    lists = [(d0, tf0), (d1, rng.integers(1, 4, size=len(d1))), (d2, rng.integers(1, 4, size=len(d2))),
             (d3, np.full(len(d3), 9, np.uint32))]
    doc_len, off, pd_, pt = _csr_corpus(rng, n_docs, lists, extra_len=20)
    T = len(lists)
    ix = m.Index(n_docs, doc_len, T, off, pd_, pt)
    oix = _PrefixOracle(orc.OracleIndex(orc.Corpus(n_docs, doc_len, T, off, pd_, pt)), max(KS))
    qs = [[0, 1], [0, 1, 2], [0, 1, 2, 3], [0, 3], [1, 2, 3]]
    _both_paths(m, ix, oix, qs, "seeds held twice")
    q_off, q_terms = _queries(qs)
    _set(ix, prune=0, **SEEDED)
    res = ix.search_batch(q_off, q_terms, 128)
    for i in range(len(qs)):
        n = int(res["n"][i])
        assert len(np.unique(res["doc"][i, :n])) == n, f"q{i}: a document appears twice"
    ix.close()
