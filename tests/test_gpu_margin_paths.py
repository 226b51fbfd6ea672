"""The f32 filter's margin kEps on the kernel instantiations test_gpu_margins.py does not reach.

Every case is a util_filter.near_threshold_case corpus (document B beats the k-th entry A, but B's f32 filter score is
below f32_rd(S_A), so a kernel built with kEps = 0 drops B) run on one instantiation of k_search_ring, and each states
where it runs: the term-count class M of its query, the pool capacity KP its limit k selects, the seeded kernel's hit-list
rows (RCfg::HCAP, 0 where the class scores each verification pass right away), the index options that select the launch
flavour, and the launches of the batch.  The restatements below (launch_ring_k, RCfg, the hand-back and suspend tests of
the kernel) check those claims against the fixture, so a case that silently moved to another instantiation fails here.

  seeded, hit list       2 terms and 3 terms at k = 10 (KP 64: 32 and 22 rows), 3 and 4 terms at k = 33 and 128 (KP 256:
                         32 rows).  B goes through the hit list and is scored by a flush, after the threshold has moved.
  seeded, no hit list    2 terms at k = 64; the 8-term class (6 and 8 terms) at k = 10 and 100.
  seeded, dense window   seed_dense_div = 0 keeps a dense query in the seeded kernel: B's window is summed from posting
                         words read from HBM (doc-id-only rings).
  two-phase resume       the suspend launch hands the query over before B's dense window; the resume launch (doc-id
                         rings) sums it.  Also the two-phase path at k = 128 (KP 256).
  hand-back              the seeded launch hands every query back (each list is longer than n_docs / seed_dense_div); the
                         RING_HANDBACK launch scores B.
  plain                  k = 224 (the last KP 256 limit), 225 and 1024 (the first and last limits of the 2048-entry shared
                         pool); the 16- and 32-term classes with B in a dense window.

The GPU test runs each with pruning on and off and demands the oracle's rows bit for bit (B among them).  The fixture check
needs no GPU: the model says kEps alone decides, and the oracle ranks B in the top k and A at k + 1 with the model's
scores."""
import numpy as np
import pytest

import util_filter as uf
from util_lib import gpu_library, set_options  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import KERNEL_PATHS, compare

CLASSES = (1, 2, 3, 4, 8, 16, 32, 64)  # bm25x_batch_prepare: a query of n live terms runs in the first class >= n
CHAMP_L = 128                          # BM25X_CHAMP_L: the seeded launch takes limits up to the champion-list length
SUSPEND_MIN = 4096                     # BM25X_SUSPEND_MIN: postings left when a two-phase query is handed over

SEEDED = dict(KERNEL_PATHS["seeded"], seed_max_terms=8)
HANDBACK = dict(SEEDED, seed_prune_min=0, seed_dense_div=0xFFFFFFFF)  # every list is "dense": all queries go back

# name: (near_threshold_case arguments, flavour, index options, class M, KP, hit-list rows, launches)
CASES = {
    "seeded_2_hits": (dict(m=1, k=10, n_docs=1000000), "seeded", SEEDED, 2, 64, 32, 2),
    "seeded_3_hits": (dict(m=2, k=10, n_docs=1000000), "seeded", SEEDED, 3, 64, 22, 2),
    "seeded_3_k33": (dict(m=2, k=33, n_docs=1000000), "seeded", SEEDED, 3, 256, 32, 2),
    "seeded_3_k128": (dict(m=2, k=128, n_docs=1000000), "seeded", SEEDED, 3, 256, 32, 2),
    "seeded_4_k33": (dict(m=3, k=33, n_docs=1000000), "seeded", SEEDED, 4, 256, 32, 2),
    "seeded_4_k128": (dict(m=3, k=128, n_docs=1000000), "seeded", SEEDED, 4, 256, 32, 2),
    "seeded_2_k64": (dict(m=1, k=64, n_docs=1000000), "seeded", SEEDED, 2, 256, 0, 2),
    "seeded_6_k10": (dict(m=5, k=10, n_docs=1000000), "seeded", SEEDED, 8, 64, 0, 2),
    "seeded_6_k100": (dict(m=5, k=100, n_docs=1000000), "seeded", SEEDED, 8, 256, 0, 2),
    "seeded_8_k10": (dict(m=7, k=10, n_docs=1000000), "seeded", SEEDED, 8, 64, 0, 2),
    "seeded_8_k100": (dict(m=7, k=100, n_docs=1000000), "seeded", SEEDED, 8, 256, 0, 2),
    "seeded_dense": (dict(m=3, k=10, n_docs=60000, binade=8.0, dense=True), "seeded", SEEDED, 4, 64, 0, 2),
    "resume_dense": (dict(m=3, k=10, n_docs=60000, binade=8.0, dense=True), "twophase", KERNEL_PATHS["twophase"], 4, 64, 0, 2),
    "twophase_k128": (dict(m=3, k=128, n_docs=1000000), "twophase", KERNEL_PATHS["twophase"], 4, 256, 0, 2),
    "handback": (dict(m=3, k=10, n_docs=1000000), "handback", HANDBACK, 4, 64, 0, 2),
    "plain_k224": (dict(m=3, k=224, n_docs=1000000), "plain", KERNEL_PATHS["plain"], 4, 256, 0, 1),
    "plain_k225": (dict(m=3, k=225, n_docs=1000000), "plain", KERNEL_PATHS["plain"], 4, 2048, 0, 1),
    "plain_k1024": (dict(m=3, k=1024, n_docs=1000000), "plain", KERNEL_PATHS["plain"], 4, 2048, 0, 1),
    "plain_16_dense": (dict(m=15, k=10, n_docs=60000, binade=8.0, dense=True), "plain", KERNEL_PATHS["plain"], 16, 64, 0, 1),
    "plain_32_dense": (dict(m=31, k=10, n_docs=60000, binade=8.0, dense=True), "plain", KERNEL_PATHS["plain"], 32, 64, 0, 1),
}


def term_class(n):
    return next(c for c in CLASSES if c >= n)


def hit_rows(M, KP):
    """RCfg<M, KP, RING_SEEDED>::HCAP: the hit list takes what the 128-byte rounding of the warp's shared-memory area
    leaves, up to 32 rows of (M + 1) words, and exists only with room for 16 rows or more."""
    R = 1 << 9                          # BM25X_DOCRING_LOG_R: doc ids per run
    map_bytes = 1 << (11 if M <= 4 else 13)
    lcap = 4 * (32 * 4) + 64            # TMAX trips of 32 lanes × 4 doc ids, + 64
    off_cand = M * R * 4 + map_bytes + KP * 16
    sst = 32 if KP <= 64 else 128
    off_hit = ((off_cand + lcap * 2 + 7) & ~7) + M * sst * 8
    smem = 227 * 1024 - 1024
    warps = min(20, smem // ((off_hit + 8 + 127) & ~127))
    rows = min(32, (((smem // warps) & ~127) - (off_hit + 24)) // ((M + 1) * 4))
    return rows if rows >= 16 else 0


def _suspends_before_b(c):
    """Two-phase, pruning off: once Sk = S_A, no term's best posting reaches Flo (every wlim is infinite) and the postings
    left are those of the dense block and B, >= BM25X_SUSPEND_MIN — the suspend launch hands the query over there."""
    Flo, _ = uf.thresholds(c["S_a"])
    left = len(c["tf_b"]) * (c["n_docs"] - c["dense_from"])
    return all(u < float(Flo) for u in c["ubd"]) and left >= SUSPEND_MIN


_FIXTURES = {}


def _case(orc, name):
    if name not in _FIXTURES:
        _FIXTURES[name] = uf.near_threshold_case(orc, **CASES[name][0], hit_rows=CASES[name][5])
    return _FIXTURES[name]


def _oracle(orc, c):
    return orc.OracleIndex(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"],
                                      k1=2.0, b=0.0))


def _where(name, c):
    """The instantiation the case claims, checked against the restated dispatch."""
    args, flavour, opts, M, KP, hcap, launches = CASES[name]
    k = c["k"]
    assert term_class(len(c["query"])) == M
    assert uf.pool_capacity(k) == KP
    if flavour in ("seeded", "handback"):
        assert 2 <= M <= 8 and k <= CHAMP_L and hit_rows(M, KP) == hcap
        for prune in (1, 0):
            assert uf.hands_back(c, opts, prune) == (flavour == "handback"), prune
    else:
        assert hcap == 0
    if flavour == "twophase":
        assert 2 <= M <= 4 and k <= 224
        if args.get("dense"):
            assert _suspends_before_b(c)
    assert launches == (2 if flavour != "plain" else 1)
    return k


@pytest.mark.parametrize("name", list(CASES))
def test_margin_path_fixture(orc, name):
    """CPU: the case runs where it says, kEps alone decides B's fate in the model (with the pruned set at Sk = S_A too,
    for the classes of <= 8 lanes), and the oracle ranks B in the top k and A right behind it with the model's scores."""
    c = _case(orc, name)
    k = _where(name, c)
    assert c["a_doc"] < c["b_doc"] and c["S_a"] < c["S_b"] and c["S_late"] < c["S_a"]
    assert c["tight"] and c["keeps"] and c["max_keps"] is not None and c["max_keps"] < uf.KEPS
    if c["m"] + 1 <= 8:
        assert c["tight_pruned"] and c["keeps_pruned"]
    hcap = CASES[name][5]
    assert len(c["late"]) == uf.late_count(k, 40, hcap) >= uf.cut_trigger(k, uf.pool_capacity(k), True) - k + hcap
    od, os_, _ = _oracle(orc, c).search_exhaustive(c["query"], k + 1)
    assert c["b_doc"] in od[:k].tolist() and od[k] == c["a_doc"]
    assert os_[k] == c["S_a"] and os_[od.tolist().index(c["b_doc"])] == c["S_b"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_margin_keeps_b_on_every_instantiation(m, orc, name):
    c = _case(orc, name)
    k = _where(name, c)
    opts, launches = CASES[name][2], CASES[name][6]
    ix = m.Index(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"], k1=2.0, b=0.0)
    oix = _oracle(orc, c)
    q_off = np.array([0, len(c["query"])], np.uint32)
    first = None
    for prune in (1, 0):
        set_options(ix, prune=prune, **opts)
        res = ix.search_batch(q_off, c["query"], k)
        assert res["stats"].launches == launches
        assert c["b_doc"] in res["doc"][0, :k].tolist(), f"{name} prune={prune}: B dropped by the filter"
        compare(res, oix, q_off, c["query"], k, what=f"{name} prune={prune}")
        if first is None:
            first = res
        else:
            assert np.array_equal(res["doc"], first["doc"]) and np.array_equal(res["score64"], first["score64"])
    ix.close()
