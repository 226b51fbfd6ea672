"""CPU: the error budget of the search kernel's f32 filter (DESIGN.md §5), checked on util_filter's restatement of it.

Per term, the f32 filter score (tf · s0f) · rcp(tf + s1f) is within TERM_BOUND_U · 2^-24 (relative) of Cache::evaluate in
f64, for k1 in {1.2, 2.0}, b in {0, 0.75, 1}, all 256 fieldnorms, tf from 1 to 2^24 − 1 and s0 over df 1 … 10^6 of 10^6
documents.  A sequential f32 sum of m positive terms adds at most (m − 1) · 2^-24, the probe loop two more additions; for
the widest sum (32 lanes) the total stays below the kernel's margin kEps = 2^-18.  The near-threshold fixtures of
test_gpu_margins.py are checked here too: in the exact regime the model is a point, its S is the oracle's score bit for
bit, and kEps alone decides B's fate."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import util_filter as uf
from test_gpu_margins import CASES

KB = [(k1, b) for k1 in (1.2, 2.0) for b in (0.0, 0.75, 1.0)]


def _tfs():
    edge = [1, 2, 3, 6, 14, 30, 255, 256, (1 << 19) - 1, 1 << 19, (1 << 23) - 1, 1 << 23, (1 << 24) - 2, (1 << 24) - 1]
    return np.unique(np.concatenate([edge, np.unique(np.logspace(0, np.log10((1 << 24) - 1), 400).astype(np.int64))]))


@pytest.mark.parametrize("k1,b", KB, ids=[f"k1={a}_b={b}" for a, b in KB])
def test_term_error_within_bound(orc, k1, b):
    L = orc.lib()
    N = 1000000
    df = np.unique(np.concatenate([[1, 2, 3, N // 2, N - 1, N], np.logspace(0, 6, 60).astype(np.int64)]))
    s0d, s1d = uf.cache(orc, N, df, k1, b, avgdl=37.5)
    tf = _tfs()
    worst = 0.0
    s1c = (C.c_double * 256)(*s1d)
    for i, s0 in enumerate(s0d):
        T, FN = np.meshgrid(tf, np.arange(256), indexing="ij")
        S = uf.score64(T, s0, s1d[FN])
        p, rl, rh = uf.term_f32(T, np.float32(s0), s1d.astype(np.float32)[FN])
        lo = (p * rl).astype(np.float64)
        hi = (p * rh).astype(np.float64)
        worst = max(worst, float(np.max(np.maximum(np.abs(lo - S), np.abs(hi - S)) / S)))
        if i % 16 == 0:  # numpy's f64 restatement is the C Cache::evaluate
            for t, f in ((1, 0), (30, 17), ((1 << 24) - 1, 255)):
                assert uf.score64(t, s0, s1d[f]) == L.orc_cache_evaluate(s0, s1c, f, t)
    assert worst < uf.TERM_BOUND_U * uf.U, worst / uf.U


def test_budget_closes_below_keps():
    """Stated bounds: the widest f32 sum of one pass (32 lanes; two-pass queries sum each group alone) and the probe loop
    of the <= 8-lane classes (8 lanes + blk_ub + rest) stay below kEps = 2^-18 = 64 · 2^-24."""
    assert uf.budget_u(uf.MAX_STREAMED) * uf.U < uf.KEPS
    assert uf.budget_u(8, uf.PROBE_EXTRA) * uf.U < uf.KEPS


@pytest.mark.parametrize("k1,b", [(1.2, 0.75), (2.0, 1.0)])
def test_sum_error_within_budget(orc, k1, b):
    """Random documents of 1 … 32 held lanes (random tf, fieldnorm, s0): the model's F interval, ascending order and the
    probe order, lies within budget_u(m) · 2^-24 · S of the f64 S."""
    rng = np.random.default_rng(5)
    N = 200000
    s0d, s1d = uf.cache(orc, N, rng.integers(1, N, size=64), k1, b, avgdl=40.0)
    for _ in range(400):
        m = int(rng.integers(1, 33))
        q = uf.Query(rng.choice(s0d, size=m, replace=False), s1d)
        tfs = rng.integers(1, 50, size=m) * (rng.random(m) < 0.8)
        tfs[0] = max(tfs[0], 1)
        fns = rng.integers(0, 256, size=m)
        S = q.exact(tfs, fns)
        held = int((tfs > 0).sum())
        for order in (None, list(rng.permutation(m))):
            lo, hi = q.filter_score(tfs, fns, order)
            err = max(abs(float(lo) - S), abs(float(hi) - S)) / S
            assert err < uf.budget_u(held) * uf.U, (m, err / uf.U)


def test_exact_regime_is_a_point(orc):
    """b = 0, k1 = 2: s1 = 2 for every fieldnorm; tf + 2 a power of two makes the reciprocal exact, so F is one value
    (p · 2^-n, the same fused or not); for other tfs the interval is two ulps wide."""
    s0d, s1d = uf.cache(orc, 100000, [7, 300, 5000], 2.0, 0.0)
    assert np.all(s1d == 2.0)
    q = uf.Query(s0d, s1d)
    for tf in uf.EXACT_TF:
        lo, hi = q.filter_score([tf] * 3)
        assert lo == hi
        assert float(uf.term_f32(tf, q.s0f[0], np.float32(2.0))[1]) == 1.0 / (tf + 2)
    lo, hi = q.filter_score([3, 3, 3])
    assert lo < hi


@pytest.mark.parametrize("name", list(CASES))
def test_near_threshold_fixtures_are_tight(orc, name):
    """Each GPU margin case: S_A < S_B with A first; F_B exact and below f32_rd(S_A) (kEps = 0 drops B) but not below
    f32_rd(S_A · (1 − 2^-18)) (the shipped kernel keeps B); and the model's S_A, S_B are the oracle's scores bit for bit."""
    args = CASES[name][0]
    c = uf.near_threshold_case(orc, **args)
    assert c["a_doc"] < c["b_doc"] and c["S_a"] < c["S_b"]
    assert c["tight"] and c["keeps"] and c["max_keps"] is not None and c["max_keps"] < uf.KEPS
    if c["m"] + 1 <= 8 and not args.get("n_rare"):
        assert c["tight_pruned"] and c["keeps_pruned"]
    oix = orc.OracleIndex(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"],
                                     k1=2.0, b=0.0))
    od, os_, _ = oix.search_exhaustive(c["query"], c["k"] + 1)
    assert od[c["k"]] == c["a_doc"] and os_[c["k"]] == c["S_a"]
    assert os_[od.tolist().index(c["b_doc"])] == c["S_b"]


def test_sass_reciprocal_and_accumulation():
    """The premise of the exact regime, read from the built library: the search kernels take the reciprocal with MUFU.RCP
    and accumulate with FMUL / FADD or FFMA (no division, no f64 in the filter sum)."""
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vectorchord-bm25_b200", "libbm25x.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(so) or not os.path.exists(tool):
        pytest.skip("needs the built library and cuobjdump")
    sass = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    funcs = sass.split("Function : ")
    ring = [f for f in funcs if "k_search_ring" in f.split("\n", 1)[0]]
    assert ring
    for f in ring:
        assert "MUFU.RCP " in f
        assert "FFMA" in f or "FMUL" in f
