"""GPU: the document-sharded index (bm25x_sharded_*) against the unsharded index built from the same corpus.  Every
comparison covers every output array (doc, score, score64, payload, n) over all nq·k rows, the slots past n included:
sharding must not change a bit."""
import threading

import numpy as np
import pytest

from util_corpora import ADVERSARIAL_BOUNDS, PARITY_CONFIGS, SHARDED_PATHS, TWO_PASS, adversarial_corpus, corpus_dict
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import ROWS, live_queries, query_csr, same_rows

pytestmark = pytest.mark.gpu



def _both(ix, sx, q_off, q_terms, k, allow=None, what=""):
    want = ix.search_batch(q_off, q_terms, k, allow=allow, want_payload=True)
    got = sx.search_batch(q_off, q_terms, k, allow=allow, want_payload=True)
    same_rows(got, want, what)
    return got, want


def _default_bounds(post_doc, n_docs, n_shards):
    """The balanced split, restated: c_d = distinct terms of document d; b_s is the smallest d > b_{s-1} with
    Σ_{d' < d} c_{d'} >= ceil(s·P/S), clamped so that every shard keeps at least one document."""
    cum = np.zeros(n_docs + 1, np.int64)
    cum[1:] = np.cumsum(np.bincount(post_doc, minlength=n_docs))
    P, S = int(cum[-1]), n_shards
    b = [0]
    for s in range(1, S):
        target = -(-s * P // S)
        d = b[-1] + 1 + int(np.searchsorted(cum[b[-1] + 1:], target, side="left"))
        b.append(min(d, n_docs - (S - s)))
    return np.array(b + [n_docs], np.uint32)


@pytest.mark.parametrize("cfg", PARITY_CONFIGS, ids=[c["name"] for c in PARITY_CONFIGS])
def test_parity_shapes_every_shard_count(m, cfg):
    c = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    q_off, q_terms = m.synth_queries(cfg["seed"] + 1000, cfg["nq"], cfg["vocab"], cfg["tmin"], cfg["tmax"],
                                     c.post_off, cfg["zipf"])
    ix = m.Index.from_corpus(c)
    for S in (1, 2, 3, 8, 16):
        sx = m.ShardedIndex.from_corpus(c, n_shards=S)
        bounds = sx.doc_bounds()
        assert np.array_equal(bounds, _default_bounds(c.post_doc, c.n_docs, S)), (S, bounds)
        info, winfo = sx.info(), ix.info()
        for f in ("n_docs", "n_terms", "n_postings", "sum_doc_len", "avgdl", "k1", "b", "device"):
            assert getattr(info, f) == getattr(winfo, f), (S, f)
        assert info.n_blocks >= winfo.n_blocks and info.device_bytes > 0
        for k in (1, 10, 100, 1000):
            _both(ix, sx, q_off, q_terms, k, what=f"{cfg['name']} S={S} k={k}")
        sx.close()
    ix.close()


def test_default_bounds_skewed_corpus(m):
    """Documents of very different lengths: the balanced split follows the postings, not the document count."""
    c = m.synth_corpus(61, 30000, 2000, 1, 400, 0.8)
    for S in (2, 5, 16):
        sx = m.ShardedIndex.from_corpus(c, n_shards=S)
        b = sx.doc_bounds()
        assert np.array_equal(b, _default_bounds(c.post_doc, c.n_docs, S))
        per = np.diff(np.searchsorted(np.sort(c.post_doc), b.astype(np.int64)))
        assert per.max() - per.min() <= 2 * 400, per   # within about one document's postings
        sx.close()


def test_adversarial_bounds(m):
    """A one-document shard, bounds off multiples of 8, a shard where every query term has local df 0, a shard holding
    all postings of a term, a shard with no postings at all — with and without a prefilter bitmap."""
    c, rng = adversarial_corpus()
    N = c["n_docs"]
    bounds = ADVERSARIAL_BOUNDS
    ix = m.Index(**c)
    sx = m.ShardedIndex(**c, n_shards=len(bounds) - 1, doc_bounds=bounds)
    assert np.array_equal(sx.doc_bounds(), bounds)
    qs = [[60], [61], [60, 61], [60, 3, 7], [61, 5], [1, 2, 3, 4], [9], [60, 61, 0, 1, 2, 3, 4, 5, 6]]
    qs += [list(rng.choice(62, size=int(rng.integers(1, 9)), replace=False)) for _ in range(40)]
    q_off, q_terms = query_csr(qs)
    allow = np.packbits(rng.random(N) < 0.4, bitorder="little")
    for k in (1, 7, 100, 300, 1025):
        for al in (None, allow):
            _both(ix, sx, q_off, q_terms, k, allow=al, what=f"adversarial k={k} allow={al is not None}")
    sx.close()
    ix.close()


def test_limits_across_the_pool_classes(m):
    c = m.synth_corpus(22, 30000, 5000, 16, 96, 1.0)
    q_off, q_terms = m.synth_queries(1022, 24, 5000, 1, 8, c.post_off, 1.0)
    ix = m.Index.from_corpus(c)
    sx = m.ShardedIndex.from_corpus(c, n_shards=3, doc_bounds=[0, 9999, 20003, 30000])
    for k in (1, 10, 100, 128, 129, 224, 225, 1000, 1024, 1025, 65535):
        _both(ix, sx, q_off, q_terms, k, what=f"k={k}")
    sx.close()
    ix.close()


@pytest.mark.parametrize("zipf", [0.0, 1.0], ids=["uniform", "zipf"])
def test_every_kernel_path_with_and_without_prefilter(m, zipf):
    c = m.synth_corpus(81, 80000, 400 if zipf == 0.0 else 4000, 6, 40, zipf)
    q_off, q_terms = m.synth_queries(82, 160, c.n_terms, 1, 8, c.post_off, zipf)
    allow = np.packbits(np.random.default_rng(9).random(c.n_docs) < 0.5, bitorder="little")
    ix = m.Index.from_corpus(c)
    sx = m.ShardedIndex.from_corpus(c, n_shards=4)
    for name, opts in SHARDED_PATHS.items():
        for idx in (ix, sx):
            for o in ("seed", "twophase", "prune"):
                idx.set_option(o, {"seed": 1, "twophase": 0, "prune": 1}[o])
            idx.set_option("seed_dense_div", 64)
            idx.set_option("seed_prune_min", 32768)
            for o, v in opts.items():
                idx.set_option(o, v)
        for k in (10, 128, 224):
            for al in (None, allow):
                _both(ix, sx, q_off, q_terms, k, allow=al, what=f"{name} k={k} allow={al is not None}")
    with pytest.raises(m.Bm25xError) as e:
        sx.set_option("no-such-option", 1)
    assert e.value.code == 1 and "unknown option" in str(e.value)
    sx.close()
    ix.close()


def test_33_to_64_terms_split_differs_per_shard(m):
    cfg = TWO_PASS[0]
    c = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    ix = m.Index.from_corpus(c)
    df = ix.df()
    rng = np.random.default_rng(11)
    counts = list(range(33, 65)) * 2
    q_off, q_terms = live_queries(rng, df, counts)
    bounds = np.array([0, 6001, 13007, c.n_docs], np.uint32)
    sx = m.ShardedIndex.from_corpus(c, n_shards=3, doc_bounds=bounds)
    # the rarest-32 group of a query by each shard's local df differs from the whole index's on some queries
    local = [np.array([np.count_nonzero((c.post_doc[c.post_off[t]:c.post_off[t + 1]] >= lo) &
                                        (c.post_doc[c.post_off[t]:c.post_off[t + 1]] < hi)) for t in range(c.n_terms)])
             for lo, hi in zip(bounds[:-1], bounds[1:])]
    differs = 0
    for i in range(len(counts)):
        q = q_terms[q_off[i]:q_off[i + 1]].tolist()
        g = lambda d: set(sorted([t for t in q if d[t] > 0], key=lambda t: (d[t], t))[:32])
        differs += any(g(ld) != g(df) for ld in local)
    assert differs > len(counts) // 2, differs
    allow = np.packbits(rng.random(c.n_docs) < 0.3, bitorder="little")
    for k in (1, 10, 225, 1025):
        for al in (None, allow):
            _both(ix, sx, q_off, q_terms, k, allow=al, what=f"33..64 terms k={k}")
    sx.close()
    ix.close()


def test_exact_ties_across_shard_boundaries_b0(m):
    """b = 0 and tf = 1 everywhere: every document holding the same query terms has exactly the same score, so result
    rows are long tie groups that cross the shard bounds; the tie order is the global doc id."""
    rng = np.random.default_rng(5)
    N = 3000
    lists = [(np.sort(rng.choice(N, size=int(rng.integers(50, 900)), replace=False)), None) for _ in range(30)]
    lists = [(d, np.ones(len(d), np.uint32)) for d, _ in lists]
    c = corpus_dict(N, lists)
    ix = m.Index(**c, b=0.0)
    bounds = [0, 333, 1001, 1002, 2222, N]
    sx = m.ShardedIndex(**c, b=0.0, n_shards=5, doc_bounds=bounds)
    qs = [list(rng.choice(30, size=int(rng.integers(1, 4)), replace=False)) for _ in range(50)]
    q_off, q_terms = query_csr(qs)
    crossing = 0
    for k in (5, 100, 1000):
        got, _ = _both(ix, sx, q_off, q_terms, k, what=f"b=0 ties k={k}")
        for i in range(len(qs)):
            n = int(got["n"][i])
            s, d = got["score64"][i, :n], got["doc"][i, :n].astype(np.int64)
            shard = np.searchsorted(bounds, d, side="right")
            crossing += int(np.sum((s[1:] == s[:-1]) & (shard[1:] != shard[:-1])))
    assert crossing > 100, crossing


def test_refusals_match_the_unsharded_index(m):
    c = m.synth_corpus(31, 3000, 100, 4, 40, 0.0)
    ix = m.Index.from_corpus(c)
    sx = m.ShardedIndex.from_corpus(c, n_shards=3)
    q_off, q_terms = m.synth_queries(32, 10, 100, 1, 4, c.post_off)
    big = np.arange(65, dtype=np.uint32)            # 65 live terms in the whole index
    cases = [(q_off, q_terms, 0), (q_off, q_terms, m.MAX_K + 1),
             (np.array([0, 3, 68], np.uint32), np.r_[np.uint32([1, 2, 3]), big], 10),
             (np.array([0, 2, 1], np.uint32), np.uint32([1, 2]), 10)]

    def refused(qo, qt, k, calls=1):
        errs = []
        for idx in (ix, sx):
            for _ in range(calls):
                with pytest.raises(m.Bm25xError) as e:
                    idx.search_batch(qo, qt, k)
                errs.append((e.value.code, str(e.value)))
        assert len(set(errs)) == 1, errs
        return errs[0]

    for qo, qt, k in cases:
        refused(qo, qt, k)

    def batch(nq, seed, big_at=(), backwards_at=()):
        qo, qt = m.synth_queries(seed, nq, 100, 1, 4, c.post_off)
        qs = [list(qt[qo[i]:qo[i + 1]]) for i in range(nq)]
        for i in big_at:
            qs[i] = list(big)
        qo, qt = query_csr(qs)
        for i in backwards_at:
            qo[i + 1] = qo[i] - 1
        return qo, qt

    # a sliced batch (4 slices of 16) whose only bad query, 40, is query 8 of the third slice
    for idx in (ix, sx):
        idx.set_option("slice_min", 16)
    assert refused(*batch(64, 33, big_at=[40]), 10) == (4, "bm25x error 4: bm25x_batch_prepare: query 8 has 65 live terms > 64")
    assert refused(*batch(64, 33, backwards_at=[40]), 10) == (1, "bm25x error 1: bm25x_batch_prepare: q_off not monotone at 8")
    # 8192 queries in one piece, canonicalised by several threads in chunks of 1024: with bad queries in several chunks the
    # message names the highest-numbered one, call after call
    for idx in (ix, sx):
        idx.set_option("slice_min", 0)
    assert refused(*batch(8192, 34, big_at=[1500, 7000], backwards_at=[4200]), 10, calls=3) == \
        (4, "bm25x error 4: bm25x_batch_prepare: query 7000 has 65 live terms > 64")
    assert refused(*batch(8192, 34, big_at=[1500, 4200], backwards_at=[7000]), 10, calls=3) == \
        (1, "bm25x error 1: bm25x_batch_prepare: q_off not monotone at 7000")
    # 65 live terms spread so that no shard sees more than 64 of them: still refused
    sx2 = m.ShardedIndex.from_corpus(c, n_shards=16)
    with pytest.raises(m.Bm25xError) as e:
        sx2.search_batch(np.array([0, 65], np.uint32), big, 10)
    assert e.value.code == 4 and "65 live terms" in str(e.value)
    sx2.close()
    sx.close()
    ix.close()


def test_lookup_terms_and_explicit_payload(m):
    """16-byte keys resolve to the segment's ordinals as on the unsharded index; an explicit payload travels with each
    shard's slice of the documents."""
    c = m.synth_corpus(31, 3000, 100, 4, 40, 0.0)
    rng = np.random.default_rng(2)
    keys = np.unique(rng.integers(1, 255, size=(c.n_terms * 2, 16), dtype=np.uint8), axis=0)[:c.n_terms]
    payload = rng.integers(0, 65535, size=(c.n_docs, 3)).astype(np.uint16)
    ix = m.Index.from_corpus(c, term_keys=keys, payload=payload)
    sx = m.ShardedIndex.from_corpus(c, n_shards=3, doc_bounds=[0, 1001, 1999, c.n_docs], term_keys=keys, payload=payload)
    probe = np.concatenate([keys[::7], np.zeros((1, 16), np.uint8), keys[-1:]])
    got = sx.lookup_terms(probe)
    assert np.array_equal(got, ix.lookup_terms(probe)) and got[-2] == m.TERM_MISSING
    assert np.array_equal(got[:-2], np.arange(0, c.n_terms, 7))
    q_off, q_terms = m.synth_queries(32, 40, 100, 1, 4, c.post_off)
    for k in (3, 50):
        _both(ix, sx, q_off, q_terms, k, what=f"payload k={k}")
    plain = m.ShardedIndex.from_corpus(c, n_shards=2)
    with pytest.raises(m.Bm25xError) as e:
        plain.lookup_terms(probe)
    assert e.value.code == 1 and "without term keys" in str(e.value)
    plain.close()
    sx.close()
    ix.close()


def test_stats_identities(m):
    c = m.synth_corpus(71, 60000, 3000, 24, 96, 1.0)
    q_off, q_terms = m.synth_queries(72, 200, 3000, 1, 8, c.post_off, 1.0)
    q_off = np.r_[q_off, q_off[-1] + 1].astype(np.uint32)       # one query without a live term
    q_terms = np.r_[q_terms, np.uint32(m.TERM_MISSING)]
    ix = m.Index.from_corpus(c)
    sx = m.ShardedIndex.from_corpus(c, n_shards=4)
    for prune in (1, 0):
        for idx in (ix, sx):
            idx.set_option("prune", prune)
            idx.set_option("twophase", 0)
        got, want = _both(ix, sx, q_off, q_terms, 10, what=f"stats prune={prune}")
        g, w = got["stats"], want["stats"]
        assert g.queries == w.queries == len(q_off) - 2
        assert g.postings == w.postings
        assert g.launches > w.launches and g.kernel_ms > 0
        if prune == 0:
            assert g.postings_fetched == w.postings_fetched == w.postings
    sx.close()
    ix.close()


def test_eight_threads_on_one_sharded_index(m):
    c = m.synth_corpus(22, 30000, 5000, 16, 96, 1.0)
    ix = m.Index.from_corpus(c)
    sx = m.ShardedIndex.from_corpus(c, n_shards=3)
    work = []
    for t in range(8):
        q_off, q_terms = m.synth_queries(500 + t, 64, 5000, 1, 8, c.post_off, 1.0)
        k = (5, 10, 100, 300)[t % 4]
        work.append((q_off, q_terms, k, ix.search_batch(q_off, q_terms, k, want_payload=True)))
    errors = []

    def run(t):
        try:
            q_off, q_terms, k, want = work[t]
            for _ in range(4):
                same_rows(sx.search_batch(q_off, q_terms, k, want_payload=True), want, f"thread {t}")
        except Exception as e:  # noqa: BLE001 — reported below
            errors.append(e)

    th = [threading.Thread(target=run, args=(t,)) for t in range(8)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors[0]
    sx.close()
    ix.close()


def test_sample_against_the_oracle(m, orc):
    c = m.synth_corpus(0xB25C0DE1, 1000, 1000, 32)
    q_off, q_terms = m.synth_queries(0xB25C0DE1 + 1000, 100, 1000, 1, 5, c.post_off)
    sx = m.ShardedIndex.from_corpus(c, n_shards=5)
    oix = orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf))
    for k in (10, 100):
        res = sx.search_batch(q_off, q_terms, k)
        for i in range(len(q_off) - 1):
            od, os_, _ = oix.search_exhaustive(q_terms[q_off[i]:q_off[i + 1]], k)
            n = int(res["n"][i])
            assert n == len(od) and np.array_equal(res["doc"][i, :n], od), (k, i)
            assert np.array_equal(res["score64"][i, :n], os_), (k, i)
            assert np.array_equal(res["score"][i, :n], os_.astype(np.float32)), (k, i)
    sx.close()


def _constructed_rows(rng, S, nq, k, levels):
    """Per shard: n <= k rows in canonical order with scores from a few levels (equal scores in every shard)."""
    rows, bases, base = [], [], 0
    for s in range(S):
        span = int(rng.integers(k + 1, 3 * k + 2))
        r = dict(doc=np.full((nq, k), 0xFFFFFFFF, np.uint32), score=np.zeros((nq, k), np.float32),
                 score64=np.zeros((nq, k)), payload=np.zeros((nq, k, 3), np.uint16), n=np.zeros(nq, np.uint32))
        for q in range(nq):
            n = int(rng.integers(0, k + 1)) if rng.random() < 0.7 else k
            sc = rng.choice(levels, size=n)
            docs = rng.choice(span, size=n, replace=False)
            order = np.lexsort((docs, -sc))                  # canonical: score desc, then doc asc
            r["doc"][q, :n], r["score64"][q, :n] = docs[order], sc[order]
            r["score"][q, :n] = sc[order].astype(np.float32)
            r["payload"][q, :n] = rng.integers(0, 65535, size=(n, 3))
            r["n"][q] = n
        rows.append(r)
        bases.append(base)
        base += span
    return rows, bases


def test_merge_kernel_against_a_fold_of_the_host_merge(m):
    rng = np.random.default_rng(17)
    for S, nq, k, levels in [(2, 50, 10, [1.0, 2.0, 3.0]), (3, 40, 100, [0.5, 0.75]), (16, 20, 33, [4.0, 4.0, 2.5]),
                             (5, 30, 1, [1.0, 2.0]), (16, 2, 65535, [1.0, 1.5, 2.0, 7.0]), (1, 10, 50, [1.0, 3.0])]:
        rows, bases = _constructed_rows(rng, S, nq, k, np.array(levels))
        got, ms = m.merge_shards(rows, bases, k)
        assert ms >= 0.0
        acc = dict(rows[0])
        acc["doc"] = np.where(np.arange(k)[None, :] < acc["n"][:, None], acc["doc"] + np.uint32(bases[0]), acc["doc"])
        for s in range(1, S):
            acc = m.merge_topk(acc, rows[s], bases[s], k)
        for key in ROWS:
            assert np.array_equal(got[key], acc[key]), (S, nq, k, key)
        assert np.array_equal(got["n"], np.minimum(sum(r["n"].astype(np.int64) for r in rows), k))


def test_shards_on_two_devices(m):
    if m.device_count() < 2:
        pytest.skip("one CUDA device visible: shards on two devices not exercised")
    c = m.synth_corpus(22, 30000, 5000, 16, 96, 1.0)
    q_off, q_terms = m.synth_queries(1022, 200, 5000, 1, 8, c.post_off, 1.0)
    ix = m.Index.from_corpus(c)
    sx = m.ShardedIndex.from_corpus(c, n_shards=3, devices=[0, 1, 1])
    allow = np.packbits(np.random.default_rng(1).random(c.n_docs) < 0.5, bitorder="little")
    for k in (10, 100, 1025):
        for al in (None, allow):
            _both(ix, sx, q_off, q_terms, k, allow=al, what=f"two devices k={k}")
    sx.close()
    ix.close()
