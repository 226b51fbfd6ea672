"""GPU: the search paths and index invariants the corpus-shape parity tests do not reach — every term-count class in one
batch, candidate pools in HBM (limit 1025 .. 65 535), seeded launches of 5..8 terms, non-default k1 / b with exact ties
at the champion-list cut, k-th / (k+1)-th scores a few ulps apart, and the index arrays (postings, blocks, score tables,
score bounds) against a CPU restatement.  Bar as test_gpu_parity: doc ids, ranks and f64 scores bit-exact against
OracleIndex.search_exhaustive, f32 scores = (float) f64 scores, unused rows 0xFFFFFFFF.  Two-pass (33..64-term) queries:
test_gpu_parity.py::test_more_than_32_terms_two_passes."""
import numpy as np
import pytest

import _pkg
from test_gpu_parity import _compare, _csr_corpus, _live_queries, _oracle_index, _PrefixOracle, _rows_identical
from test_gpu_zz_growing import _expect, _setup
from util_index import assert_matches, read_back, restate

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


# kernel paths of the 2..8-term classes, as index options (a seeded launch that keeps every query: no hand-back)
PATHS = dict(seeded=dict(seed=1, twophase=0, seed_prune_min=0xFFFFFFFF, seed_dense_div=0),
             twophase=dict(seed=0, twophase=1),
             plain=dict(seed=0, twophase=0))


def _set(ix, **opts):
    for name, value in opts.items():
        ix.set_option(name, value)


def test_class_boundary_matrix_sliced(m, orc):
    """One batch mixing every term-count class boundary (1, 2, 3, 4 | 5, 8 | 9, 16 | 17, 32 | 33, 64 live terms) plus
    queries without a live term, in shuffled order: bm25x_batch_prepare groups and scatters them per class.  One piece and
    cut into slices: the same rows, equal to the oracle."""
    c = m.synth_corpus(201, 20000, 1500, 8, 120, 0.0)
    ix = m.Index.from_corpus(c)
    rng = np.random.default_rng(201)
    counts = [1, 2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 64] * 6
    q_off, q_terms = _live_queries(rng, ix.df(), counts)
    qs = [q_terms[q_off[i]:q_off[i + 1]] for i in range(len(counts))] + [np.zeros(0, np.uint32),
                                                                          np.array([m.TERM_MISSING, 10 ** 7], np.uint32)]
    qs = [qs[i] for i in rng.permutation(len(qs))]
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    q_terms = np.concatenate(qs).astype(np.uint32)
    oix = _PrefixOracle(_oracle_index(orc, c), 100)
    for k in (10, 100):
        ix.set_option("slice_min", 0)
        one = ix.search_batch(q_off, q_terms, k, want_payload=True)
        ix.set_option("slice_min", 8)  # 74 queries: 9 slices
        cut = ix.search_batch(q_off, q_terms, k, want_payload=True)
        assert cut["stats"].launches > one["stats"].launches
        _rows_identical(one, cut, f"sliced k={k}")
        assert np.array_equal(one["payload"], cut["payload"])
        _compare(one, oix, q_off, q_terms, k, what=f"class matrix k={k}")
    ix.close()


def test_limits_above_1024_hbm_pools(m, orc):
    """Limits beyond 1024 keep their candidate pools in HBM (KP = 131072: per-warp slices of a scratch buffer, bitonic
    sort in global memory, cut lazily at KP - 32).  160k documents over 50 terms: the 3- and 8-term queries match more than
    65 535 documents, so even the largest pool is cut; single-term queries (~39k documents) fill it only partly.  Scratch per
    launch = CTAs x warps x KP x 16 B, and a class of 3 queries fills one CTA: well under 100 MB here."""
    c = m.synth_corpus(211, 160000, 50, 4, 24, 0.0)
    ix = m.Index.from_corpus(c)
    df = ix.df()
    rng = np.random.default_rng(211)
    counts = [1, 3, 8] * 3
    q_off, q_terms = _live_queries(rng, df, counts)
    allow = np.packbits(rng.random(c.n_docs) < 0.6, bitorder="little")
    keep = np.unpackbits(allow, bitorder="little")[:c.n_docs].astype(bool)

    def matches(i, al):
        docs = np.unique(np.concatenate([c.post_doc[c.post_off[t]:c.post_off[t + 1]] for t in q_terms[q_off[i]:q_off[i + 1]]]))
        return len(docs) if al is None else int(keep[docs].sum())

    hits = [matches(i, None) for i in range(len(counts))]
    assert max(hits) > 65535 > min(hits), hits
    assert max(matches(i, allow) for i in range(len(counts))) > 65535
    ks = (1024, 1025, 5000, 65535)
    oix = _PrefixOracle(_oracle_index(orc, c), max(ks))
    for k in ks:
        for al in (None, allow):
            ix.set_option("prune", 1)
            on = ix.search_batch(q_off, q_terms, k, allow=al)
            ix.set_option("prune", 0)
            off = ix.search_batch(q_off, q_terms, k, allow=al)
            _rows_identical(on, off, f"prune on/off k={k} allow={al is not None}")
            _compare(on, oix, q_off, q_terms, k, allow=al, what=f"hbm pool k={k} allow={al is not None}")
    ix.set_option("prune", 1)
    ix.close()


def test_growing_segment_limit_2000(m, orc):
    """Sealed + growing search at a limit of the HBM-pool class: both top-2000 lists and their merge."""
    sealed, g, ix, gix, oix = _setup(m, orc, 63, 3000, 3000, 60, 5, 1.0)
    N = sealed.n_docs
    q_off, q_terms = m.synth_queries(1063, 24, 60, 1, 8, sealed.post_off, 1.0)
    both = ix.search_batch_growing(gix, q_off, q_terms, 2000)
    cut = 0
    for i in range(len(q_off) - 1):
        ed, es = _expect(oix, g, N, q_terms[q_off[i]:q_off[i + 1]], 2000)
        n = int(both["n"][i])
        assert n == len(ed) and both["doc"][i, :n].tolist() == ed, f"q{i} merged ids"
        assert both["score64"][i, :n].tolist() == es, f"q{i} merged f64 scores"
        assert np.array_equal(both["score"][i, :n], np.array(es).astype(np.float32)), f"q{i} merged f32 scores"
        assert np.all(both["doc"][i, n:] == 0xFFFFFFFF)
        cut += n == 2000
    assert cut >= 5
    gix.close()
    ix.close()


def test_seeded_5_to_8_terms(m, orc):
    """Queries of 5..8 terms run seeded by default (seed_max_terms 8) when their lists are sparse: on this corpus no
    list reaches n_docs / seed_dense_div or seed_prune_min postings, so no query is handed back.  Seeded 8-term launches,
    the 4-term maximum (plain kernel for the class) and seeding off return the same bits; a sample is checked against the
    oracle."""
    c = m.synth_corpus(221, 200000, 20000, 8, 40, 0.0)
    ix = m.Index.from_corpus(c)
    df = ix.df()
    q_off, q_terms = m.synth_queries(222, 200, c.n_terms, 5, 8, c.post_off, 0.0)
    n_live = np.diff(q_off)
    assert n_live.min() == 5 and n_live.max() == 8
    assert int(df[q_terms].max()) < min(c.n_docs // 64, 32768)  # the default hand-back thresholds
    oix = _PrefixOracle(_oracle_index(orc, c), 129)
    for k in (1, 10, 127, 128, 129):
        got = {}
        for name, opts in dict(seed8=dict(seed=1, seed_max_terms=8), seed4=dict(seed=1, seed_max_terms=4),
                               off=dict(seed=0, seed_max_terms=8)).items():
            for prune in (1, 0):
                _set(ix, prune=prune, **opts)
                got[name, prune] = ix.search_batch(q_off, q_terms, k)
        for key, res in got.items():
            _rows_identical(res, got["off", 1], f"{key} k={k}")
        # one class (8) in the batch: a seeded launch and the launch of its hand-back list, else one launch
        assert got["seed8", 1]["stats"].launches == (2 if k <= 128 else 1)
        assert got["seed4", 1]["stats"].launches == 1
        _compare(got["seed8", 1], oix, q_off[:41], q_terms, k, what=f"seeded 5..8 k={k}")
    ix.close()


KB = [(1.2, 0.0), (2.0, 1.0), (2.0, 0.75)]


@pytest.mark.parametrize("k1,b", KB, ids=[f"k1={a}_b={b}" for a, b in KB])
def test_k1_b_edges(m, orc, k1, b):
    """Non-default BM25 parameters (the reference accepts k1 in [1.2, 2.0], b in [0, 1]): seeded, two-phase and plain
    kernels agree with each other and with the oracle built with the same k1 / b."""
    c = m.synth_corpus(231, 30000, 1500, 4, 80, 0.6)
    ix = m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=k1, b=b)
    info = ix.info()
    assert (info.k1, info.b) == (k1, b)
    oix = _PrefixOracle(orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf,
                                                   k1=k1, b=b)), 1000)
    q_off, q_terms = m.synth_queries(232, 120, c.n_terms, 1, 8, c.post_off, 0.6)
    for k in (1, 10, 128, 129, 224, 1000):
        got = {}
        for name, opts in PATHS.items():
            for prune in (1, 0):
                _set(ix, prune=prune, **opts)
                got[name, prune] = ix.search_batch(q_off, q_terms, k)
        for key, res in got.items():
            _rows_identical(res, got["plain", 1], f"{key} k={k}")
        _compare(got["seeded", 1], oix, q_off, q_terms, k, what=f"k1={k1} b={b} k={k}")
    ix.close()


def test_b0_tie_flood_at_champion_cut(m, orc):
    """b = 0: the fieldnorm drops out of the score, so postings with the same tf tie exactly whatever their norm (distinct
    tie signatures, one score).  Term 0 is held with tf = 1 by 1500 documents, so its champion list (128) ends inside one
    tie group; term 2 has 60 tf = 2 postings ahead of its tie group.  Paired with a rare term, at limits around 128."""
    rng = np.random.default_rng(241)
    n_docs = 4000
    d2 = np.sort(rng.choice(n_docs, size=860, replace=False))
    tf2 = np.ones(860, np.uint32)
    tf2[rng.choice(860, size=60, replace=False)] = 2
    lists = [(np.sort(rng.choice(n_docs, size=1500, replace=False)), np.ones(1500, np.uint32)),
             (np.sort(rng.choice(n_docs, size=40, replace=False)), rng.integers(1, 4, size=40)),
             (d2, tf2)]
    for _ in range(3):  # filler terms: document lengths (norms) vary
        d = np.sort(rng.choice(n_docs, size=2500, replace=False))
        lists.append((d, rng.integers(1, 7, size=len(d))))
    doc_len, off, pd_, pt = _csr_corpus(rng, n_docs, lists, extra_len=300)
    T = len(lists)
    for k1 in (1.2, 2.0):
        ix = m.Index(n_docs, doc_len, T, off, pd_, pt, k1=k1, b=0.0)
        oix = _PrefixOracle(orc.OracleIndex(orc.Corpus(n_docs, doc_len, T, off, pd_, pt, k1=k1, b=0.0)), 1001)
        qs = [[0], [0, 1], [2, 1], [0, 2], [0, 1, 2], [0, 3], [2, 4, 1]]
        q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
        q_terms = np.array([t for q in qs for t in q], dtype=np.uint32)
        for k in (127, 128, 129, 1000):
            got = {}
            for name in ("seeded", "plain"):
                for prune in (1, 0):
                    _set(ix, prune=prune, **PATHS[name])
                    got[name, prune] = ix.search_batch(q_off, q_terms, k)
            for key, res in got.items():
                _rows_identical(res, got["plain", 1], f"{key} k1={k1} k={k}")
            _compare(got["seeded", 1], oix, q_off, q_terms, k, what=f"tie flood k1={k1} k={k}")
            if k < 1000:  # the cut is inside a tie group: the last row of [0, 1] ties with rows it excludes
                assert got["plain", 1]["score64"][1, k - 1] == oix.search_exhaustive(qs[1], k + 1)[1][k]
        ix.close()


def test_near_ties_at_the_kth_score(m, orc):
    """The f32 filter rejects a document only below Sk * (1 - 2^-18): a (k+1)-th score a few ulps under the k-th must
    never push the k-th out.  For each query, the ranks i of the oracle's full ranking where the relative gap
    0 < (s[i-1] - s[i]) / s[i] < 2^-17, then the GPU at limit k = i on every kernel path, pruning on and off."""
    c = m.synth_corpus(251, 20000, 300, 1, 300, 0.0)  # lists of ~5000 postings: crowded scores, thousands of near ties
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    q_off, q_terms = m.synth_queries(252, 300, c.n_terms, 1, 6, c.post_off, 0.0)
    ranking, cases = {}, []
    for qi in range(len(q_off) - 1):
        q = q_terms[q_off[qi]:q_off[qi + 1]]
        od, os_, _ = oix.search_exhaustive(q, c.n_docs)
        ranking[qi] = (od, os_)
        s = os_[:1025]
        gap = (s[:-1] - s[1:]) / s[1:]
        for i in np.flatnonzero((gap > 0) & (gap < 2.0 ** -17)) + 1:
            cases.append((float(gap[i - 1]), qi, int(i)))
    cases.sort()
    assert len(cases) >= 200 and cases[20][0] < 2.0 ** -22, (len(cases), cases[:21])  # not vacuous: ulp-close pairs
    cases = cases[:400]  # the closest pairs
    by_k = {}
    for _, qi, k in cases:
        by_k.setdefault(k, []).append(qi)

    for k, qis in sorted(by_k.items()):
        sub_off = np.cumsum([0] + [int(q_off[i + 1] - q_off[i]) for i in qis]).astype(np.uint32)
        sub_terms = np.concatenate([q_terms[q_off[i]:q_off[i + 1]] for i in qis]).astype(np.uint32)
        first = None
        for name, opts in PATHS.items():
            for prune in (1, 0):
                _set(ix, prune=prune, **opts)
                res = ix.search_batch(sub_off, sub_terms, k)
                if first is None:
                    first = res
                    for j, qi in enumerate(qis):
                        od, os_ = ranking[qi]
                        n = int(res["n"][j])
                        assert n == k, (qi, k, n)
                        assert np.array_equal(res["doc"][j], od[:k]), f"q{qi} k={k}: ids"
                        assert np.array_equal(res["score64"][j], os_[:k]), f"q{qi} k={k}: f64 scores"
                        assert np.array_equal(res["score"][j], os_[:k].astype(np.float32)), f"q{qi} k={k}: f32 scores"
                else:
                    _rows_identical(res, first, f"near tie k={k} {name} prune={prune}")
    ix.close()


@pytest.mark.parametrize("shape", ["varlen", "b0"])
def test_index_arrays_match_cpu_restatement(m, orc, shape):
    """The 13 device arrays of an index (Index.layout(), read back with cudaMemcpy) and its derived ones against the CPU
    restatement of tests/util_index.py (numpy and the oracle's C Cache / fieldnorm): postings with the fieldnorm folded in and their pad slots, offsets, block descriptors, score
    tables bit-equal, and the score bounds pruning trusts — ubd = (best single-posting score) x (1 + 2^-40) and blk_ub =
    the smallest f32 >= (block max) x (1 + 2^-40), bit-exact, each >= every posting score it bounds."""
    if shape == "varlen":
        c, k1, b = m.synth_corpus(21, 20000, 3000, 1, 300, 0.0), 1.2, 0.75
    else:
        c, k1, b = m.synth_corpus(261, 20000, 2000, 1, 200, 0.8), 1.2, 0.0
    ix = m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=k1, b=b)
    oix = orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=k1, b=b))
    L = orc.lib()
    r = restate(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, k1, b, doc_len=c.doc_len)
    lay = ix.layout()
    assert lay.avgdl == oix.avgdl
    assert np.array_equal(r.fieldnorm, [L.orc_index_fieldnorm(oix.h, d) for d in range(c.n_docs)])
    der = ix.derived()
    assert_matches(read_back(lay, der), lay, der, r, f"create {shape}")
    # what pruning relies on: no posting scores above its block's bound, no block maximum above its term's bound
    blk_of = np.repeat(np.arange(r.n_blocks), np.diff(np.append(r.blk_start, r.n_postings)))
    assert np.all(r.blk_ub[blk_of].astype(np.float64) >= r.score)
    assert np.all(r.ubd[r.blk_term] >= r.block_max) and np.all(r.ubd[r.term] >= r.score)
    ix.close()
