"""GPU: the f32 filter's safety margin kEps (bm25x_search_ring.cuh refresh_filter) is load-bearing on every kernel path:
a kernel built with kEps = 0 fails every case of this module.

Each case is a corpus built by util_filter.near_threshold_case: document A is the k-th entry once the pool has been cut
with A and the better documents in it (whichever order a kernel verifies the early candidates in, later low-scoring
documents overflow the pool again before B), a later document B has the larger exact score, and B's f32 filter score is below f32_rd(S_A) — exactly, because the
corpus lies in the exact regime (b = 0, k1 = 2, tf + 2 a power of two).  A kernel whose margin were 0 would drop B; the
shipped kernel must return the oracle's rows bit for bit (ids, ranks, f64 scores, f32 scores = (float) f64 scores), with
pruning on and off.  Pruning lowers the streamed threshold by the pruned bounds, so with pruning on the margin decides
only through the probe loop's last test (Fres against FloT, classes of <= 8 lanes): the model asserts that too where it
applies, and the 16- / 32-lane classes and two-pass queries claim non-vacuity with pruning off only.

The other margins are covered by kEps (DESIGN.md §5): each adds at most a few f32 ulps (2^-24 relative) of error
against a budget of 2^-18 − (8 + 31)·2^-24 that kEps leaves over after the worst filter error.
  - FloT / Flo rounded down (_rd): _rn moves the threshold up by at most half an ulp of Sk, 2^-24·Sk.
  - ne_prefix_f rounded up: _rn lowers `rest` by at most half an ulp, < 2^-24·Sk (rest <= ALPHA·Sk).
  - blk_ub rounded up and inflated by 2^-40: _rd lowers one bound by less than one ulp (2^-23 of a term's score).
  - ctf shrunk by 2^-20: the one-compare single-term test solves F >= Flo for tf; a document with S >= Sk needs a tf at
    least kEps·s0 / (s0 − Flo) >= 2^-18 (relative) above the solved value, far more than the s1f / ctf roundings (2^-23).
  - ub_oth · (1 + 1e-12): covers the butterfly sum of <= 32 f64 bounds (< 2^-47 relative), and ubd is inflated by 2^-40
    already; against the f32 threshold it is 2^-18·Sk that decides.
So none of these alone changes a result while kEps = 2^-18; they matter only together with a margin near 0."""
import numpy as np
import pytest

import _pkg
from test_gpu_parity import _compare
from test_gpu_paths import PATHS, _set
import util_filter as uf

pytestmark = pytest.mark.gpu

# name: (near_threshold_case arguments, kernel path options, launches of the batch's one class)
CASES = {
    "plain_6_lanes": (dict(m=5, k=10, n_docs=1000000), PATHS["plain"], 1),    # class 8, KEEPW verification
    "class_16": (dict(m=15, k=10, n_docs=1000000), PATHS["plain"], 1),        # filter_term loop
    "class_32": (dict(m=31, k=10, n_docs=1000000), PATHS["plain"], 1),
    "seeded_4_lanes": (dict(m=3, k=10, n_docs=1000000), PATHS["seeded"], 2),  # seeded launch + (empty) hand-back launch
    "two_phase": (dict(m=3, k=10, n_docs=1000000), PATHS["twophase"], 2),     # suspend launch, resume launch (doc ids) finds B
    "two_pass": (dict(m=8, k=10, n_docs=1000000, n_rare=32), PATHS["plain"], 1),  # 41 lanes: B holds group 1 only
    "dense_window": (dict(m=4, k=10, n_docs=60000, binade=8.0, dense=True), PATHS["plain"], 1),
    "hbm_pool": (dict(m=3, k=1025, n_docs=1000000), PATHS["plain"], 1),       # k = 1025: pool in HBM, lazy cut
}


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


@pytest.mark.parametrize("name", list(CASES))
def test_margin_keeps_the_later_better_document(m, orc, name):
    args, opts, launches = CASES[name]
    c = uf.near_threshold_case(orc, **args)
    k = c["k"]
    assert c["tight"] and c["keeps"], "the model says kEps alone decides"
    assert c["a_doc"] < c["b_doc"] and c["S_a"] < c["S_b"]
    if c["m"] + 1 <= 8 and not args.get("n_rare"):
        assert c["tight_pruned"] and c["keeps_pruned"], "the model says kEps decides in the probe loop too"
    ix = m.Index(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"], k1=2.0, b=0.0)
    info = ix.info()
    assert (info.k1, info.b) == (2.0, 0.0)
    oix = orc.OracleIndex(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"],
                                     k1=2.0, b=0.0))
    q_off = np.array([0, len(c["query"])], np.uint32)
    od, os_, _ = oix.search_exhaustive(c["query"], k + 1)
    # the oracle's ranking: B in the top k, A right behind it at k + 1, with the scores the model computed
    assert c["b_doc"] in od[:k].tolist() and od[k] == c["a_doc"]
    assert os_[k] == c["S_a"] and os_[od.tolist().index(c["b_doc"])] == c["S_b"]
    first = None
    for prune in (1, 0):
        _set(ix, prune=prune, **opts)
        res = ix.search_batch(q_off, c["query"], k)
        assert res["stats"].launches == launches
        _compare(res, oix, q_off, c["query"], k, what=f"{name} prune={prune}")
        if first is None:
            first = res
        else:
            assert np.array_equal(res["doc"], first["doc"]) and np.array_equal(res["score64"], first["score64"])
    ix.close()
