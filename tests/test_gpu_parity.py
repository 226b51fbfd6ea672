"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.
Bar: doc ids / ranks bit-exact under the canonical tie rule, f64 scores bit-exact, f32 scores = (float) f64 scores
(the kernel writes out_score = (float) score64, the merge copies it)."""
import os

import numpy as np
import pytest

import _pkg
from util_parity import check_topk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


def _oracle_index(orc, c):
    return orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf))


def _compare(res, oix, q_off, q_terms, k, allow=None, what=""):
    for i in range(len(q_off) - 1):
        q = q_terms[q_off[i]:q_off[i + 1]]
        od, os_, _ = oix.search_exhaustive(q, k, allow=allow)
        n = int(res["n"][i])
        assert n == len(od), f"{what} q{i}: n {n} != {len(od)}"
        assert np.array_equal(res["doc"][i, :n], od), f"{what} q{i} k{k}: ids\n got {res['doc'][i, :n]}\nwant {od}"
        assert np.array_equal(res["score64"][i, :n], os_), f"{what} q{i}: f64 scores not bit-exact"
        assert np.array_equal(res["score"][i, :n], os_.astype(np.float32)), f"{what} q{i}: f32 scores"
        assert np.all(res["doc"][i, n:] == 0xFFFFFFFF)


class _PrefixOracle:
    """OracleIndex.search_exhaustive at one large limit, memoised per (query, bitmap): the canonical order (score desc,
    doc asc) is total, so the top-k of every smaller k is a prefix of it."""

    def __init__(self, oix, kmax):
        self.oix, self.kmax, self.memo = oix, kmax, {}

    def search_exhaustive(self, q, k, allow=None):
        assert k <= self.kmax
        q = np.ascontiguousarray(q, dtype=np.uint32)
        key = (q.tobytes(), None if allow is None else np.asarray(allow).tobytes())
        if key not in self.memo:
            self.memo[key] = self.oix.search_exhaustive(q, self.kmax, allow=allow)
        od, os_, tg = self.memo[key]
        return od[:k], os_[:k], tg


def _live_queries(rng, df, counts, weighted=False):
    """One query per entry of `counts` with exactly that many distinct terms of df > 0, ascending ids.  weighted: terms
    drawn in proportion to df (head terms in most queries)."""
    live = np.flatnonzero(df > 0)
    p = df[live] / df[live].sum() if weighted else None
    qs = [np.sort(rng.choice(live, size=n, replace=False, p=p)) for n in counts]
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    return q_off, np.concatenate(qs).astype(np.uint32)


def _rows_identical(a, b, what):
    for key in ("doc", "score", "score64", "n"):
        assert np.array_equal(a[key], b[key]), f"{what}: {key}"


def _csr_corpus(rng, n_docs, lists, extra_len=0):
    """Term-major CSR from explicit posting lists [(doc ids, tfs)]; a document's length is its Σ tf plus up to
    `extra_len` tokens of terms outside the corpus (varied norms)."""
    off = np.zeros(len(lists) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d, _ in lists])
    post_doc = np.concatenate([np.asarray(d, np.uint32) for d, _ in lists])
    post_tf = np.concatenate([np.asarray(t, np.uint32) for _, t in lists])
    doc_len = np.bincount(post_doc, weights=post_tf, minlength=n_docs).astype(np.uint32)
    if extra_len:
        doc_len += rng.integers(0, extra_len + 1, size=n_docs).astype(np.uint32)
    return doc_len, off, post_doc, post_tf


TWO_PASS = [
    # uniform vocabulary: df is not monotone in the term id, so the two groups interleave in id order
    dict(name="uniform", seed=101, n=20000, vocab=1500, lmin=8, lmax=120, zipf=0.0, weighted=False),
    # dense: 72 terms, long documents (dense windows in pass 0)
    dict(name="dense", seed=102, n=4000, vocab=72, lmin=60, lmax=400, zipf=0.5, weighted=False),
    # Zipf, terms drawn by df: head terms pruned while group 1 is probed
    dict(name="zipf", seed=103, n=30000, vocab=3000, lmin=16, lmax=96, zipf=1.0, weighted=True),
]


@pytest.mark.parametrize("cfg", TWO_PASS, ids=[c["name"] for c in TWO_PASS])
def test_more_than_32_terms_two_passes(m, orc, cfg):
    """33..64 live terms run as two passes of the 32-term kernel: the host puts the 32 rarest terms (by df, then id) first,
    pass 0 streams them and probes the others, pass 1 streams the others and keeps only documents without a group-0 term,
    and the exact f64 sum merges both groups back into ascending term order.  Bit-exact against the oracle for every
    limit class, pruning on and off, with and without a prefilter bitmap, plain and two-phase options."""
    c = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    ix = m.Index.from_corpus(c)
    df = ix.df()
    rng = np.random.default_rng(cfg["seed"])
    counts = [33, 40, 48, 63, 64] * 3
    q_off, q_terms = _live_queries(rng, df, counts, weighted=cfg["weighted"])
    assert np.array_equal(np.diff(q_off), counts)
    if cfg["name"] == "uniform":  # the (df, id) split is not a cut in id order
        inter = 0
        for i in range(len(counts)):
            q = q_terms[q_off[i]:q_off[i + 1]]
            g0 = sorted(q.tolist(), key=lambda t: (df[t], t))[:32]
            inter += max(g0) > min(set(q.tolist()) - set(g0))
        assert inter == len(counts)
    allow = np.packbits(rng.random(c.n_docs) < 0.3, bitorder="little")
    ks = (1, 10, 100, 225, 1000, 1025)
    oix = _PrefixOracle(_oracle_index(orc, c), max(ks))
    for k in ks:
        for al in (None, allow):
            first = None
            for two in (0, 1):
                for prune in (1, 0):
                    ix.set_option("twophase", two)
                    ix.set_option("prune", prune)
                    res = ix.search_batch(q_off, q_terms, k, allow=al)
                    if first is None:
                        first = res
                        _compare(res, oix, q_off, q_terms, k, allow=al, what=f"{cfg['name']} k={k} allow={al is not None}")
                    else:
                        _rows_identical(res, first, f"{cfg['name']} k={k} twophase={two} prune={prune}")
    ix.close()


def test_more_than_32_terms_rarest_split_ties_and_refusals(m, orc):
    """The rarest-32 split when many terms share the df at the 32/33 boundary (the term id decides), raw queries of 80
    terms that reduce to <= 64 live ones (duplicates, unknown ids, TERM_MISSING: the canonical query's rows), and the
    refusal of 65 live terms (BM25X_ERR_UNSUPPORTED)."""
    rng = np.random.default_rng(7)
    n_docs, T = 3000, 80
    want_df = np.array([40] * 16 + [90] * 30 + list(rng.integers(200, 900, size=T - 46)))
    want_df = want_df[rng.permutation(T)]  # the boundary terms sit anywhere in id order
    lists = [(np.sort(rng.choice(n_docs, size=int(d), replace=False)), rng.integers(1, 5, size=int(d))) for d in want_df]
    doc_len, off, pd_, pt = _csr_corpus(rng, n_docs, lists, extra_len=50)
    ix = m.Index(n_docs, doc_len, T, off, pd_, pt)
    oix = orc.OracleIndex(orc.Corpus(n_docs, doc_len, T, off, pd_, pt))
    assert np.array_equal(ix.df(), want_df)
    rare, tied, common = (np.flatnonzero(want_df == 40), np.flatnonzero(want_df == 90), np.flatnonzero(want_df >= 200))
    qs = [np.concatenate([rare, tied, common[:18]]),                    # 64: the split cuts the df = 90 group at 16 of 30
          np.concatenate([rare[:6], tied, common[:4]]),                 # 40: 26 of the 30 tied terms in group 0
          np.concatenate([tied, common[:10]])]                          # 40: group 0 = the 30 tied + 2 common terms
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    q_terms = np.concatenate([np.sort(q) for q in qs]).astype(np.uint32)
    for k in (1, 10, 100, 1000, 1025):
        for prune in (1, 0):
            ix.set_option("prune", prune)
            _compare(ix.search_batch(q_off, q_terms, k), oix, q_off, q_terms, k, what=f"tie split k={k} prune={prune}")
    ix.set_option("prune", 1)

    # 80 raw terms, <= 64 live: the same rows as the canonical query
    c = m.synth_corpus(104, 8000, 600, 8, 64, 0.0)
    cix = m.Index.from_corpus(c)
    df = cix.df()
    live = np.flatnonzero(df > 0)
    raws, canon = [], []
    for n_live in (33, 60, 64):
        q = rng.choice(live, size=n_live, replace=False)
        junk = [m.TERM_MISSING] * 4 + [c.n_terms, c.n_terms + 7, 10 ** 6] + list(rng.choice(q, size=80 - n_live - 7))
        raw = rng.permutation(np.concatenate([q, np.array(junk)]).astype(np.uint32))
        assert len(raw) == 80
        raws.append(raw)
        canon.append(np.sort(q).astype(np.uint32))
    r_off = np.cumsum([0] + [len(q) for q in raws]).astype(np.uint32)
    c_off = np.cumsum([0] + [len(q) for q in canon]).astype(np.uint32)
    c_terms = np.concatenate(canon)
    for k in (10, 1025):
        a = cix.search_batch(r_off, np.concatenate(raws), k)
        b = cix.search_batch(c_off, c_terms, k)
        _rows_identical(a, b, f"raw vs canonical k={k}")
        _compare(b, _oracle_index(orc, c), c_off, c_terms, k, what=f"canonical k={k}")
    # 65 live terms: refused for the whole batch (two passes of 32 lanes cover 64)
    q65 = np.sort(rng.choice(live, size=65, replace=False)).astype(np.uint32)
    for q in (q65, np.concatenate([q65, q65[:10], [m.TERM_MISSING]]).astype(np.uint32)):
        with pytest.raises(m.Bm25xError) as e:
            cix.search_batch(np.array([0, 3, 3 + len(q)], np.uint32), np.concatenate([q[:3], q]), 10)
        assert e.value.code == 4
    cix.close()
    ix.close()


CONFIGS = [
    dict(name="C1", seed=0xB25C0DE1, n=1000, vocab=1000, lmin=32, lmax=32, zipf=0.0, nq=100, tmin=3, tmax=3),
    dict(name="varlen", seed=21, n=20000, vocab=3000, lmin=1, lmax=300, zipf=0.0, nq=80, tmin=1, tmax=8),
    dict(name="zipf", seed=22, n=30000, vocab=5000, lmin=16, lmax=96, zipf=1.0, nq=80, tmin=1, tmax=8),
    dict(name="dense", seed=23, n=5000, vocab=40, lmin=5, lmax=400, zipf=1.1, nq=60, tmin=1, tmax=8),
    dict(name="manyterms", seed=24, n=8000, vocab=600, lmin=8, lmax=64, zipf=0.8, nq=40, tmin=9, tmax=32),
    dict(name="ties", seed=25, n=50000, vocab=200, lmin=16, lmax=16, zipf=0.0, nq=60, tmin=1, tmax=4),
]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c["name"] for c in CONFIGS])
def test_search_matches_oracle(m, orc, cfg):
    c = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    q_off, q_terms = m.synth_queries(cfg["seed"] + 1000, cfg["nq"], cfg["vocab"], cfg["tmin"], cfg["tmax"],
                                     c.post_off, cfg["zipf"])
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    for k in (1, 10, 100, 1000):
        res = ix.search_batch(q_off, q_terms, k)
        _compare(res, oix, q_off, q_terms, k, what=cfg["name"])
    ix.close()


def test_golden_sqllogictest_ranking(m, orc, golden):
    from test_oracle_golden import _slt_corpus
    for ids, want in [(list(range(1, 11)), golden["ranking_full_index"]), ([2, 4, 6, 8, 10], golden["ranking_even_ids"]),
                      ([1, 3, 5, 7, 9], golden["ranking_odd_ids"])]:
        c, tid = _slt_corpus(orc, golden, ids)
        ix = m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf)
        docs, scores = ix.search([tid["postgresql"]], 10)
        assert [ids[d] for d in docs] == want
        od, os_, _ = orc.OracleIndex(c).search_exhaustive([tid["postgresql"]], 10)
        assert np.array_equal(scores, os_)
        ix.close()


def test_edge_cases(m, orc):
    c = m.synth_corpus(31, 3000, 100, 4, 40, 0.0)
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    # empty query, unknown terms, duplicates, unsorted, TERM_MISSING (search.rs:55-62)
    qs = [[], [1000000], [5, 5, 9, 5], [9, 5], [m.TERM_MISSING, 7], [3]]
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    q_terms = np.array([t for q in qs for t in q], dtype=np.uint32)
    res = ix.search_batch(q_off, q_terms, 7, want_payload=True)
    _compare(res, oix, q_off, q_terms, 7, what="edge")
    assert res["n"][0] == 0 and res["n"][1] == 0
    assert np.array_equal(res["doc"][2], res["doc"][3])
    # payload default = synthetic ctid of the doc id
    d = res["doc"][5, 0]
    assert tuple(res["payload"][5, 0]) == ((d // 291) >> 16, (d // 291) & 0xFFFF, d % 291 + 1)
    # zero queries
    r0 = ix.search_batch(np.zeros(1, np.uint32), np.zeros(0, np.uint32), 5)
    assert r0["doc"].shape == (0, 5)
    # k == 0 → the reference's "number of needed rows is set to 0" error (scanners/default.rs:114-116)
    with pytest.raises(m.Bm25xError) as e:
        ix.search_batch(q_off, q_terms, 0)
    assert e.value.code == 5
    with pytest.raises(m.Bm25xError) as e:
        ix.search_batch(q_off, q_terms, m.MAX_K + 1)
    assert e.value.code == 4
    ix.close()


def test_prefilter_bitmap(m, orc):
    c = m.synth_corpus(41, 20000, 300, 8, 60, 0.9)
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    rng = np.random.default_rng(5)
    keep = rng.random(c.n_docs) < 0.2
    allow = np.packbits(keep, bitorder="little")
    q_off, q_terms = m.synth_queries(42, 40, 300, 1, 6, c.post_off, 0.9)
    res = ix.search_batch(q_off, q_terms, 25, allow=allow)
    _compare(res, oix, q_off, q_terms, 25, allow=allow, what="prefilter")
    ix.close()


def test_pruning_on_off_identical(m, orc):
    """MaxScore-style pruning (non-streamed head terms, HBM probes for candidates) must not change a single bit of the
    result; with Zipf head terms in most queries it must also stream fewer postings than the exhaustive run."""
    c = m.synth_corpus(71, 60000, 3000, 24, 96, 1.0)
    q_off, q_terms = m.synth_queries(72, 200, 3000, 2, 8, c.post_off, 1.0)
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    on = ix.search_batch(q_off, q_terms, 10)
    ix.set_option("prune", 0)
    off = ix.search_batch(q_off, q_terms, 10)
    for key in ("doc", "score", "score64", "n"):
        assert np.array_equal(on[key], off[key]), key
    _compare(on, oix, q_off, q_terms, 10, what="prune")
    if os.environ.get("BM25X_SEED_FORCE", "0") in ("", "0"):  # (a seeded launch never prunes: nothing to compare)
        assert 0 < on["stats"].postings_fetched < off["stats"].postings_fetched
    with pytest.raises(m.Bm25xError):
        ix.set_option("no-such-option", 1)
    ix.close()


@pytest.mark.parametrize("zipf", [0.0, 1.0], ids=["uniform", "zipf"])
def test_kernel_paths_identical(m, orc, zipf):
    """The three ways a 2..4-term query can run — seeded launch (champion lists + doc-id-only stream), two-phase launches
    (8-byte postings, then doc ids only), one unseeded launch — return the same bits, with pruning on and off, for limits
    around the champion-list length (128) and the two-phase limit (224); a sample is checked against the oracle."""
    c = m.synth_corpus(81, 80000, 400 if zipf == 0.0 else 4000, 6, 40, zipf)
    q_off, q_terms = m.synth_queries(82, 160, c.n_terms, 2, 4, c.post_off, zipf)
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    for k in (1, 10, 100, 128, 129, 224):
        for prune in (1, 0):
            ix.set_option("prune", prune)
            got = {}
            for name, (seed, two, spm, div) in dict(seeded=(1, 0, 1 << 30, 0), handback=(1, 0, 64, 0), dense=(1, 0, 1 << 30, 8),
                                                    twophase=(0, 1, 0, 0), plain=(0, 0, 0, 0)).items():
                ix.set_option("seed", seed)
                ix.set_option("twophase", two)
                # seeded launches hand queries back to the plain kernel: skewed ones (a list >= seed_prune_min postings and
                # 8x the shortest) and dense ones (a list of n_docs / seed_dense_div postings or more; 0: never)
                ix.set_option("seed_prune_min", spm)
                ix.set_option("seed_dense_div", div)
                got[name] = ix.search_batch(q_off, q_terms, k)
            for name in ("seeded", "handback", "dense", "twophase"):
                for key in ("doc", "score", "score64", "n"):
                    assert np.array_equal(got[name][key], got["plain"][key]), (name, key, k, prune)
        _compare(got["seeded"], oix, q_off[:25], q_terms, k, what=f"paths k={k}")
    ix.close()


def test_replica_same_device_identical(m, orc):
    """bm25x_index_get_layout / alloc_replica / finalize_replica on ONE GPU: the 13 replicated arrays copied device to
    device (what shard.replicate_index does with NCCL broadcasts), the derived structures (doc-id copy, champion lists)
    rebuilt by finalize_replica — the replica answers like the original, seeded and plain kernel."""
    from util_cuda import D2D, cudart
    rt = cudart()
    c = m.synth_corpus(95, 60000, 5000, 8, 48, 0.0)
    q_off, q_terms = m.synth_queries(96, 150, c.n_terms, 1, 8, c.post_off, 0.0)
    ix = m.Index.from_corpus(c)
    lay = ix.layout()
    rep = m.Index.alloc_replica(lay, 0)
    with pytest.raises(m.Bm25xError):  # not finalized yet
        rep.search_batch(q_off, q_terms, 10)
    rl = rep.layout()
    for i in range(len(lay.dev_ptr)):
        assert rl.bytes[i] == lay.bytes[i]
        assert rt.cudaMemcpy(rl.dev_ptr[i], lay.dev_ptr[i], lay.bytes[i], D2D) == 0
    rep.finalize_replica()
    for seed in (1, 0):
        ix.set_option("seed", seed)
        rep.set_option("seed", seed)
        for k in (10, 100):
            a, b = ix.search_batch(q_off, q_terms, k), rep.search_batch(q_off, q_terms, k)
            for key in ("doc", "score", "score64", "n"):
                assert np.array_equal(a[key], b[key]), (key, seed, k)
    _compare(b, _oracle_index(orc, c), q_off[:30], q_terms, 100, what="replica")
    rep.close()
    ix.close()


def test_broker_over_an_index_matches_direct_search(m, orc):
    """The batching broker (include/bm25x_broker.h) over a real index handle: 16 concurrent callers, limits of several
    classes — every caller gets exactly the rows of a direct search with its own limit."""
    import threading
    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    c = m.synth_corpus(97, 30000, 2000, 6, 40, 0.5)
    q_off, q_terms = m.synth_queries(98, 96, c.n_terms, 1, 6, c.post_off, 0.5)
    ix = m.Index.from_corpus(c)
    limits = [1, 10, 32, 40, 128, 300, 2000]
    want = {k: ix.search_batch(q_off, q_terms, k, want_payload=True) for k in limits}
    br = bm.Broker(index=ix, max_batch=64, max_wait_us=5000)
    got, errs = [None] * 96, []

    def client(t):
        try:
            for i in range(t, 96, 16):
                got[i] = (limits[i % len(limits)], br.search(q_terms[q_off[i]:q_off[i + 1]], limits[i % len(limits)], want_payload=True))
        except Exception as e:  # pragma: no cover
            errs.append(e)

    ts = [threading.Thread(target=client, args=(t,)) for t in range(16)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    for i, (k, (docs, s64, pay)) in enumerate(got):
        n = int(want[k]["n"][i])
        assert len(docs) == n
        assert np.array_equal(docs, want[k]["doc"][i, :n]) and np.array_equal(s64, want[k]["score64"][i, :n])
        assert np.array_equal(pay, want[k]["payload"][i, :n])
    st = br.stats()
    assert st.requests == 96 and st.batches < 96
    br.close()
    ix.close()


def test_sliced_search_batch_identical(m, orc):
    """bm25x_search_batch pipelines large batches as slices (prepare of slice s + 1 and download of slice s - 1 overlap the
    kernels of slice s): same rows as one piece, with and without a prefilter bitmap; statistics add up."""
    c = m.synth_corpus(91, 40000, 900, 4, 60, 0.6)
    q_off, q_terms = m.synth_queries(92, 333, c.n_terms, 1, 8, c.post_off, 0.6)
    ix = m.Index.from_corpus(c)
    rng = np.random.default_rng(3)
    allow = np.packbits(rng.random(c.n_docs) < 0.7, bitorder="little")
    for al in (None, allow):
        ix.set_option("slice_min", 0)
        one = ix.search_batch(q_off, q_terms, 10, allow=al, want_payload=True)
        ix.set_option("slice_min", 16)  # 16 slices of ~21 queries
        cut = ix.search_batch(q_off, q_terms, 10, allow=al, want_payload=True)
        for key in ("doc", "score", "score64", "payload", "n"):
            assert np.array_equal(one[key], cut[key]), key
        assert cut["stats"].queries == one["stats"].queries and cut["stats"].postings == one["stats"].postings
        assert cut["stats"].bytes_algo == one["stats"].bytes_algo and cut["stats"].launches >= one["stats"].launches
    _compare(cut, _oracle_index(orc, c), q_off[:30], q_terms, 10, allow=allow, what="sliced")
    ix.close()


def test_evaluate_matches_oracle_bitwise(m, orc):
    c = m.synth_corpus(51, 5000, 400, 2, 120, 0.8)
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    rng = np.random.default_rng(7)
    docs, queries = [], []
    for _ in range(300):
        nt = int(rng.integers(0, 40))
        t = np.sort(rng.choice(450, size=nt, replace=False)).astype(np.uint32)   # some ids are unknown (>= 400)
        docs.append(m.Document(t, rng.integers(1, 9, size=nt).astype(np.uint32)))
        nq = int(rng.integers(0, 9))
        queries.append(m.Query(np.sort(rng.choice(450, size=nq, replace=False)).astype(np.uint32)))
    got = ix.evaluate_batch(docs, queries)
    want = np.array([oix.evaluate(d.terms, d.tfs, q.terms) for d, q in zip(docs, queries)])
    assert np.array_equal(got, want)
    ix.close()


def test_wand_reference_path_agrees_tie_aware(m, orc):
    """The restated reference algorithm (Block-max WAND, heap tie order) vs the GPU result, tie-aware —
    the comparison a real reference run would need (SURVEY §8c)."""
    c = m.synth_corpus(61, 40000, 2000, 16, 80, 1.0)
    ix = m.Index.from_corpus(c)
    oix = _oracle_index(orc, c)
    q_off, q_terms = m.synth_queries(62, 50, 2000, 1, 8, c.post_off, 1.0)
    res = ix.search_batch(q_off, q_terms, 10)
    for i in range(50):
        q = q_terms[q_off[i]:q_off[i + 1]]
        wd, ws = oix.search_wand(q, 10)
        n = int(res["n"][i])
        check_topk(wd, ws, res["doc"][i, :n], res["score64"][i, :n], rtol=1e-12, what=f"q{i}")
    ix.close()


def test_config2_sample_1M_docs(m, orc):
    """BASELINE config 2 at full size (1M docs, vocab 30k, 64 terms/doc): 10k single-term queries top-10 on the GPU,
    a sample checked against the oracle + size-independent properties on the whole batch."""
    c = m.synth_corpus(0xB25C0DE2, 1_000_000, 30000, 64)
    q_off, q_terms = m.synth_queries(0xB25C0DE2 + 1000, 10000, 30000, 1, 1, c.post_off)
    ix = m.Index.from_corpus(c)
    res = ix.search_batch(q_off, q_terms, 10)
    assert np.all(res["n"] == 10)
    s = res["score64"]
    assert np.all(s[:, :-1] >= s[:, 1:])                                   # sortedness
    tie = s[:, :-1] == s[:, 1:]
    assert np.all(res["doc"][:, :-1][tie] < res["doc"][:, 1:][tie])        # canonical tie order
    oix = _oracle_index(orc, c)
    idx = np.arange(0, 10000, 97)
    sub_off = np.arange(len(idx) + 1, dtype=np.uint32)
    sub = {k: (v[idx] if isinstance(v, np.ndarray) else v) for k, v in res.items()}
    _compare(sub, oix, sub_off, q_terms[idx], 10, what="C2")
    ix.close()


def test_lookup_terms_16_byte_keys_then_search(m, orc):
    """address_tokens::read (crates/bm25/src/address_tokens.rs:61-98) + the skip of unknown tokens (search.rs:55-62):
    16-byte interned keys → term ordinals → search.  Short tokens are interned as their zero-padded bytes
    (crates/bm25/src/vector.rs:19-24)."""
    c = m.synth_corpus(81, 5000, 300, 8, 60, 0.5)
    words = sorted(f"tok{i:05d}".encode() for i in range(300))           # strictly ascending byte strings
    keys = np.zeros((300, 16), dtype=np.uint8)
    for i, w in enumerate(words):
        keys[i, :len(w)] = list(w)
    ix = m.Index.from_corpus(c, term_keys=keys)
    miss = np.zeros((2, 16), dtype=np.uint8)
    miss[0, :5] = list(b"nope!")                                          # sorts after every key
    miss[1, :3] = list(b"abc")                                            # sorts before every key
    look = np.concatenate([keys[[5, 17, 299, 0]], miss])
    ords = ix.lookup_terms(look)
    assert ords.tolist() == [5, 17, 299, 0, m.TERM_MISSING, m.TERM_MISSING]
    # a query in key space: unknown tokens are dropped, the rest searched — identical to the ordinal query
    q_off = np.array([0, len(ords)], dtype=np.uint32)
    res = ix.search_batch(q_off, ords, 10)
    oix = _oracle_index(orc, c)
    _compare(res, oix, np.array([0, 4], dtype=np.uint32), np.array([5, 17, 299, 0], dtype=np.uint32), 10, what="lookup")
    ix.close()
    # keys must be strictly ascending (the reference's token address tree is sorted): rejected at create
    bad = keys.copy()
    bad[[10, 11]] = bad[[11, 10]]
    with pytest.raises(m.Bm25xError) as e:
        m.Index.from_corpus(c, term_keys=bad)
    assert e.value.code == 1
    dup = keys.copy()
    dup[11] = dup[10]
    with pytest.raises(m.Bm25xError):
        m.Index.from_corpus(c, term_keys=dup)
    # an index created without keys addresses terms by ordinal only
    plain = m.Index.from_corpus(c)
    with pytest.raises(m.Bm25xError, match="without term keys"):
        plain.lookup_terms(keys[:1])
    plain.close()
