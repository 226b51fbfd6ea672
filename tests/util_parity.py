"""Search results against the CPU oracle and against each other: the queries of a batch (query_csr, live_queries),
the bit-exact comparison with the oracle's exhaustive scorer (compare, PrefixOracle), the comparison of two result dicts
(same_rows) and the kernel paths a search can be pinned to (KERNEL_PATHS).

check_topk is the tie-aware comparison of a top-k result against the canonical exhaustive oracle (SURVEY §8c):
(i) the score multiset must match within rtol; (ii) doc ids must match exactly at every rank whose
score differs from both neighbours; (iii) inside a tie group returned ids must be members of the
oracle's full tie group (checked by rescoring through `score_of`)."""
import numpy as np

ROWS = ("doc", "score", "score64", "payload", "n")

# kernel paths of the 2..8-term classes, as index options (a seeded launch that keeps every query: no hand-back)
KERNEL_PATHS = dict(seeded=dict(seed=1, twophase=0, seed_prune_min=0xFFFFFFFF, seed_dense_div=0),
                    twophase=dict(seed=0, twophase=1),
                    plain=dict(seed=0, twophase=0))


def query_csr(qs):
    """Queries as the search calls take them: (q_off, q_terms), both uint32."""
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    return q_off, np.array([t for q in qs for t in q], dtype=np.uint32)


def oracle_index(orc, c):
    return orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf))


def compare(res, oix, q_off, q_terms, k, allow=None, what=""):
    """Result rows against the oracle's exhaustive scorer: ids, ranks and f64 scores bit-exact, f32 scores = (float) f64
    scores, unused rows 0xFFFFFFFF."""
    for i in range(len(q_off) - 1):
        q = q_terms[q_off[i]:q_off[i + 1]]
        od, os_, _ = oix.search_exhaustive(q, k, allow=allow)
        n = int(res["n"][i])
        assert n == len(od), f"{what} q{i}: n {n} != {len(od)}"
        assert np.array_equal(res["doc"][i, :n], od), f"{what} q{i} k{k}: ids\n got {res['doc'][i, :n]}\nwant {od}"
        assert np.array_equal(res["score64"][i, :n], os_), f"{what} q{i}: f64 scores not bit-exact"
        assert np.array_equal(res["score"][i, :n], os_.astype(np.float32)), f"{what} q{i}: f32 scores"
        assert np.all(res["doc"][i, n:] == 0xFFFFFFFF)


class PrefixOracle:
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


def live_queries(rng, df, counts, weighted=False):
    """One query per entry of `counts` with exactly that many distinct terms of df > 0, ascending ids.  weighted: terms
    drawn in proportion to df (head terms in most queries)."""
    live = np.flatnonzero(df > 0)
    p = df[live] / df[live].sum() if weighted else None
    qs = [np.sort(rng.choice(live, size=n, replace=False, p=p)) for n in counts]
    return query_csr(qs)


def same_rows(a, b, what):
    """Two result dicts hold the same rows: every row array that either holds is in both, with the same shape and
    values."""
    for key in ROWS:
        x, y = a.get(key), b.get(key)
        if x is None and y is None:
            continue
        assert x is not None and y is not None, f"{what}: `{key}` in one result only"
        assert x.shape == y.shape, f"{what}: `{key}` shape {x.shape} != {y.shape}"
        if not np.array_equal(x, y):
            raise AssertionError(f"{what}: `{key}` differs at {np.argwhere(x != y)[:3].tolist()}")


def check_topk(docs, scores, o_docs, o_scores, rtol, score_of=None, canonical=False, what=""):
    docs = np.asarray(docs)
    scores = np.asarray(scores, dtype=np.float64)
    o_docs = np.asarray(o_docs)
    o_scores = np.asarray(o_scores, dtype=np.float64)
    assert len(docs) == len(o_docs), f"{what}: count {len(docs)} != oracle {len(o_docs)}"
    if len(docs) == 0:
        return
    assert np.all(scores[:-1] >= scores[1:] - 0.0), f"{what}: scores not descending"
    np.testing.assert_allclose(scores, o_scores, rtol=rtol, atol=0, err_msg=f"{what}: score multiset")
    if canonical:
        # bit-exact ids/ranks under the canonical rule (score desc, doc asc)
        assert np.array_equal(docs, o_docs), f"{what}: ids differ\n got {docs}\n want {o_docs}"
        return
    n = len(docs)
    for i in range(n):
        lo = o_scores[i - 1] if i > 0 else np.inf
        hi = o_scores[i + 1] if i + 1 < n else -np.inf
        tol = rtol * abs(o_scores[i])
        isolated = (lo - o_scores[i] > tol) and (o_scores[i] - hi > tol) and i + 1 < n
        if isolated:
            assert docs[i] == o_docs[i], f"{what}: rank {i} doc {docs[i]} != {o_docs[i]}"
        elif score_of is not None:
            s = score_of(int(docs[i]))
            assert abs(s - o_scores[i]) <= tol + 1e-300, f"{what}: rank {i} doc {docs[i]} not in tie group"
    assert len(set(docs.tolist())) == n, f"{what}: duplicate docs"
