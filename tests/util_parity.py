"""Tie-aware comparison of a top-k result against the canonical exhaustive oracle (SURVEY §8c):
(i) the score multiset must match within rtol; (ii) doc ids must match exactly at every rank whose
score differs from both neighbours; (iii) inside a tie group returned ids must be members of the
oracle's full tie group (checked by rescoring through `score_of`)."""
import numpy as np

ROWS = ("doc", "score", "score64", "payload", "n")


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
