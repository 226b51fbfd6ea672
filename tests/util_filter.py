"""CPU restatement of the search kernel's f32 filter (bm25x_device.cuh score_f32, bm25x_search_ring.cuh refresh_filter,
the verification branches and the probe loop of pruned terms), and the near-threshold fixtures built from it.

The kernel drops a candidate when its f32 filter score F is below f32_rd(Sk·(1 − kEps) − ub_ne − ub_oth); everything
that passes is re-scored in f64.  F per term is (tf · s0f) · rcp(tf + s1f[fn]), with s0f / s1f the host's round-to-nearest
casts of the f64 tables, summed in f32 in ascending lane (= ascending term id) order.  rcp.approx.ftz.f32 is the one
operation that cannot be restated bit for bit: it is modelled as the interval [prev(rn(1/x)), next(rn(1/x))] (PTX: at most
1 ulp), except when x is a power of two, where it is exact.  The f32 accumulation F += p·r may be contracted into an FFMA
by the compiler: the interval covers both forms.

Exact regime: b = 0 and k1 = 2.0 make s1 = 2.0 for every fieldnorm; with tf + 2 a power of two (tf in {2, 6, 14, 30, …})
the reciprocal is exact and p·r is an exact scaling, so F is one f32 value whichever form the compiler emitted."""
import ctypes as C
from fractions import Fraction

import numpy as np

from util_parity import KERNEL_PATHS

F32 = np.float32
U = 2.0 ** -24        # f32 unit roundoff
KEPS = 2.0 ** -18     # kEps of k_search_ring: reject only when F < f32_rd(Sk·(1 − kEps) − …)
ALPHA = 0.5           # BM25X_PRUNE_ALPHA
EXACT_TF = (2, 6, 14, 30)  # tf + 2 a power of two: rcp exact when s1 = 2

# Error budget (DESIGN.md §5), in units of U, relative to the exact score S:
#   one term: s0f (1) + s1f (1) + tf + s1f (1) + rcp (2: 1 ulp) + tf·s0f (1) + ·r (1), and the f64 S itself (< 2^-50)
TERM_BOUND_U = 8
MAX_STREAMED = 32     # lanes of one pass: every f32 sum has at most 32 terms (two-pass queries: per group)
PROBE_EXTRA = 2       # the probe loop's block test adds blk_ub and rest to Fres: two more f32 additions


def budget_u(m, extra=0):
    """Bound of |F − S| / S for an f32 sum of m terms (sequential, all positive: γ_(m−1+extra)) in units of U."""
    return TERM_BOUND_U + (m - 1 + extra)


def cache(orc, n_docs, df, k1, b, avgdl=1.0):
    """(s0d per df, s1d[256]) from the oracle's C Cache::new (bm25.rs:340-352)."""
    L = orc.lib()
    s1 = (C.c_double * 256)()
    s0 = np.empty(len(df))
    for i, d in enumerate(df):
        v = C.c_double()
        L.orc_cache_new(int(n_docs), int(d), float(k1), float(b), float(avgdl), C.byref(v), s1)
        s0[i] = v.value
    return s0, np.array(s1[:])


def score64(tf, s0d, s1d):
    """Cache::evaluate in f64, the reference's operation order: (tf · s0) / (tf + s1)."""
    tf = np.asarray(tf, dtype=np.float64)
    return (tf * np.asarray(s0d, np.float64)) / (tf + np.asarray(s1d, np.float64))


def sum64(vals):
    s = 0.0
    for v in vals:
        s = float(np.float64(s) + np.float64(v))
    return s


def f32_rd(x):
    """Largest f32 <= the f64 x (__double2float_rd)."""
    f = F32(x)
    return f if float(f) <= x else np.nextafter(f, F32(-np.inf))


def f32_ru(x):
    f = F32(x)
    return f if float(f) >= x else np.nextafter(f, F32(np.inf))


def rcp(x):
    """rcp.approx.f32 of the f32 array x as an interval (lo, hi): exact on powers of two, else rn(1/x) ± 1 ulp."""
    x = np.asarray(x, F32)
    r = F32(1.0) / x
    exact = np.frexp(x)[0] == 0.5
    return (np.where(exact, r, np.nextafter(r, F32(0))).astype(F32),
            np.where(exact, r, np.nextafter(r, F32(np.inf))).astype(F32))


def term_f32(tf, s0f, s1f):
    """score_f32 per term: (p, r_lo, r_hi) with p = tf·s0f rounded, F_term in [p·r_lo, p·r_hi]."""
    tff = np.asarray(tf).astype(F32)
    p = (tff * np.asarray(s0f, F32)).astype(F32)
    lo, hi = rcp(tff + np.asarray(s1f, F32))
    return p, lo, hi


def accumulate(parts, start=(F32(0), F32(0))):
    """The kernel's F += score_f32(...) over `parts` (p, r_lo, r_hi) in the given order: an interval (lo, hi).  A term
    with an exact reciprocal adds the exact product p·r (fused or not: the same value)."""
    lo, hi = start
    for p, rl, rh in parts:
        p, rl, rh = F32(p), F32(rl), F32(rh)
        if rl == rh:
            q = F32(p * rl)
            lo, hi = F32(lo + q), F32(hi + q)
            continue
        lo, hi = min(F32(lo + F32(p * rl)), _fma(p, rl, lo)), max(F32(hi + F32(p * rh)), _fma(p, rh, hi))
    return lo, hi


def _fma(a, b, c):
    """FFMA: a·b + c rounded once to the nearest f32 (ties to even)."""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    lo = f32_rd(float(x))
    if Fraction(float(lo)) > x:
        lo = np.nextafter(lo, F32(-np.inf))
    if Fraction(float(lo)) == x:
        return lo
    hi = np.nextafter(lo, F32(np.inf))
    mid = (Fraction(float(lo)) + Fraction(float(hi))) / 2
    if x != mid:
        return lo if x < mid else hi
    return lo if (int(lo.view(np.uint32)) & 1) == 0 else hi


class Query:
    """One query's terms in lane order (ascending term id within a pass) with its score tables."""

    def __init__(self, s0d, s1d):
        self.s0d = np.asarray(s0d, np.float64)
        self.s0f = self.s0d.astype(F32)
        self.s1d = np.asarray(s1d, np.float64)
        self.s1f = self.s1d.astype(F32)

    def exact(self, tfs, fns=None):
        """S of a document holding lane i with tf tfs[i] (0: not held): the oracle's f64 sum in ascending term order."""
        fns = np.zeros(len(tfs), int) if fns is None else np.asarray(fns)
        return sum64(score64(t, self.s0d[i], self.s1d[fns[i]]) for i, t in enumerate(tfs) if t)

    def parts(self, tfs, fns=None):
        fns = np.zeros(len(tfs), int) if fns is None else np.asarray(fns)
        return {i: term_f32(t, self.s0f[i], self.s1f[fns[i]]) for i, t in enumerate(tfs) if t}

    def filter_score(self, tfs, fns=None, order=None):
        """F over the held lanes in `order` (default ascending lane: every verification branch and the dense
        accumulator)."""
        parts = self.parts(tfs, fns)
        order = sorted(parts) if order is None else [i for i in order if i in parts]
        return accumulate([parts[i] for i in order])


def thresholds(Sk, ub_ne=0.0, ub_oth=0.0, keps=KEPS):
    """refresh_filter: (Flo over the streamed terms, FloT over all terms)."""
    return f32_rd(Sk * (1.0 - keps) - ub_ne - ub_oth), f32_rd(Sk * (1.0 - keps))


def pruned_lanes(ubd, Sk, ub_oth=0.0):
    """The MaxScore rule at threshold Sk: lanes leave by ascending bound (ties: lowest lane) while the sum of their bounds
    (plus ub_oth) stays <= ALPHA · Sk; one lane always stays streamed.  Returns the lanes in the order they left."""
    order = sorted(range(len(ubd)), key=lambda i: (ubd[i], i))
    out, ub_ne = [], 0.0
    for i in order[:-1]:
        if not (ub_ne + ubd[i] + ub_oth <= ALPHA * Sk):
            break
        out.append(i)
        ub_ne += ubd[i]
    return out


def probe_order(m, pruned):
    """Order in which the KEEPW classes (<= 8 lanes) sum F when terms are pruned: the streamed lanes ascending, then the
    pruned ones largest bound first (the reverse of the order they left)."""
    return [i for i in range(m) if i not in pruned] + list(reversed(pruned))


def largest_rejecting_keps(F, Sk):
    """The largest kEps = 2^-e (e = 17 … 30) at which F < f32_rd(Sk·(1 − kEps)), i.e. a kernel with that margin would drop
    a document of f32 score F against threshold Sk; None when even kEps = 0 keeps it."""
    if not F < f32_rd(Sk):
        return None
    for e in range(17, 31):
        if F < f32_rd(Sk * (1.0 - 2.0 ** -e)):
            return 2.0 ** -e
    return 0.0


def _next_up(f):
    return float(np.nextafter(F32(f), F32(np.inf)))


def pool_capacity(k):
    """KP of the launch that answers a limit of k (bm25x_search.cu launch_ring_k): the warp's candidate pool, in shared
    memory up to 2048 entries, in HBM beyond."""
    return 64 if k <= 32 else 256 if k <= 224 else 2048 if k <= 1024 else 131072


def cut_trigger(k, kp, threshold):
    """The pool size at which pool_insert cuts the pool back to k (k_search_ring): always above KP − 32 entries; before
    that, at k + 32 entries, unless the pool is a large one (KP > 128) that already has a threshold (the lazy cut)."""
    lazy = kp > 128 and threshold
    return kp - 31 if lazy else min(kp - 31, k + 32)


def late_count(k, n_low, hit_rows=0):
    """Late low documents of near_threshold_case.  A kernel may cut the pool first with A (or some high documents)
    missing; after that cut the pool holds k entries and has a threshold.  A enters, and every late low document beats
    that threshold, so once pool_insert has cut again at cut_trigger(k, KP, True) entries A is the k-th: that takes
    cut_trigger − k late documents.  The seeded kernel's hit list (hit_rows rows, RCfg::HCAP) keeps up to hit_rows − 1
    of them waiting across windows until the flush that scores B: their insertion comes after B's filter, so hit_rows
    more.  An HBM pool (KP > 2048) is cut lazily only beyond KP − 32 = 131 040 entries, more than a list here holds:
    there the cases rest on the first cut, which the n_low early low documents force at k + 32 entries.  Never fewer
    than n_low, the count the fixtures of k <= 32 without a hit list were built with."""
    kp = pool_capacity(k)
    return n_low if kp > 2048 else max(n_low, cut_trigger(k, kp, True) - k + hit_rows)


def near_threshold_case(orc, m, k, n_docs, *, binade=16.0, dense=False, n_rare=0, hit_rows=0, seed=0, tries=3000):
    """A corpus (b = 0, k1 = 2: exact regime) in which the margin kEps alone decides whether a top-k document survives.

    Query terms: ids 0 … m − 1 (B's terms), m (term x, A's knob) and, with n_rare, m + 1 … m + n_rare (df 1: the rarest,
    group 0 of a two-pass query).  Doc ids, in order: k − 1 − [n_rare > 0] "high" documents (B's terms, tf 30: above
    everything else); with n_rare, one document holding the rare terms; document A (term x at a large tf, a few of B's
    terms at tf <= 3, searched so that next_f32(F_B) <= S_A < S_B); 40 "low" documents (terms 0 and 1, tf 1); the fillers —
    single-term documents spread evenly (sparse) or, with `dense`, a block of documents holding every B term with tf 1 —
    with late_count(k, 40, hit_rows) "late low" documents (terms 0 and 1, tf 3: above every low document and filler,
    below S_A) halfway through them; and last, document B (B's m terms, tf 2).  The late low documents make the threshold S_A
    whatever order the early candidates were verified in: a kernel may cut the pool for the first time before the high
    documents or A are in it (the seeded kernel verifies its champion seeds and the documents of the lower runs first),
    and then, with nothing else above that first threshold, the k-th score would stay below S_A until B.  With them, the
    pool overflows again once A and the high documents are in, and is cut to exactly those k.  B's exact score beats S_A
    while B's f32 filter score is below f32_rd(S_A): a kernel without the margin drops B.

    B's dfs are searched among the terms whose s0 (just above `binade`) rounds down most in f32, in the order that leaves
    F_B furthest below S_B.  m = 2: B's two tfs are searched too (tf 6 or 14 where tf 2 cannot lose enough).

    m = 1 (a 2-term query): B holds term x too, so that it has two holders (a document of one holder would be a seed or a
    single-term posting).  Two terms at tf 2 cannot lose more than one f32 ulp, so B's tfs and A's tf on term 0 are
    searched as well, and term x's df is solved so that A's large tf on x lands S_A in the window (_pair_case).  Its late
    low documents hold term 0 at tf 1 and x at tf 2 (tf 3 on both would beat B)."""
    rng = np.random.default_rng(seed)
    k1, b = 2.0, 0.0
    n_high = k - 1 - (1 if n_rare else 0)
    n_low = 40
    n_late = late_count(k, n_low, hit_rows)
    # s0 = 3 ln((N + 1) / (df + 0.5)) in [binade, 1.1 binade]
    cand = np.arange(int(n_docs * np.exp(-1.1 * binade / 3)) + 1, int(n_docs * np.exp(-binade / 3)))
    s0c, s1d = cache(orc, n_docs, cand, k1, b)
    assert np.all(s1d == 2.0) and len(cand) >= 2 * m
    rel = (s0c - s0c.astype(F32).astype(np.float64)) / s0c
    if m == 1:
        assert not n_rare and not dense
        return _pair_case(orc, cand, s0c, s1d, k, n_docs, n_high, n_low, n_late, rng)
    pool = np.argsort(-rel)[:max(60, 2 * m)]
    # two terms at tf 2 lose at most one ulp of their f32 sum (each s0f / 2 is exact, the sum rounds once): with two
    # terms B's tfs are searched too (tf + 2 a power of two: 6 and 14 round tf·s0f as well)
    tfbs = [(2,) * m] if m > 2 else [(6, 6), (2, 6), (6, 2), (6, 14), (14, 6)]
    found = {}
    for _ in range(tries):
        pick = tuple(rng.choice(pool, size=m, replace=False))
        q = Query(s0c[list(pick)], s1d)
        for tfb in tfbs:
            F = float(q.filter_score(tfb)[0])
            S = q.exact(tfb)
            if S > _next_up(F):
                found[pick, tfb] = (S - _next_up(F)) / S
    for pick, tfb in sorted(found, key=lambda p: -found[p])[:40]:
        case = _with_a(orc, np.array(pick), cand, s0c, s1d, m, k, n_docs, n_high, n_low, n_late, dense, n_rare, rng,
                       list(tfb))
        if case is not None and (case["tight_pruned"] or m + 1 > 8 or n_rare):
            return case
    raise AssertionError(f"no near-threshold fixture for m={m}")


def _pair_case(orc, cand, s0c, s1d, k, n_docs, n_high, n_low, n_late, rng):
    """The 2-term fixture: B = (tf t0 on term 0, tf tx on x), A = (tf a on term 0, a large tf T on x).  With T large,
    S_A = s0_0·a/(a + 2) + s0_x·(1 − 2/(T + 2)) reaches S_B = s0_0·t0/(t0 + 2) + s0_x·tx/(tx + 2) only when
    s0_x·2/(tx + 2) is just above s0_0·(t0/(t0 + 2) − a/(a + 2)): x's df is taken from that neighbourhood, and T solved."""
    need = n_high + n_low + n_late + 16  # postings of each term: high, low, late documents, A, B and a few fillers
    cand_x = np.arange(need, n_docs // 8)
    for t0, tx, a in ((6, 2, 1), (14, 2, 1), (6, 6, 2), (14, 6, 2), (6, 2, 2), (2, 6, 1), (14, 2, 2)):
        c = t0 / (t0 + 2) - a / (a + 2)
        for i in rng.permutation(len(cand))[:400]:
            if cand[i] < need:
                continue
            s0_0 = float(s0c[i])
            target = (tx + 2) / 2 * s0_0 * c  # s0_x at which T would be infinite
            d0 = int((n_docs + 1) * np.exp(-target / 3))
            dfx = cand_x[(cand_x >= d0 - 40) & (cand_x <= d0 + 2)]
            if len(dfx) == 0:
                continue
            s0x, _ = cache(orc, n_docs, dfx, 2.0, 0.0)
            for d, s0_x in zip(dfx, s0x):
                q = Query(np.array([s0_0, s0_x]), s1d)
                F_b = float(q.filter_score([t0, tx])[0])
                S_b = q.exact([t0, tx])
                lo_w = _next_up(F_b)
                if not S_b > lo_w:
                    continue
                part = float(score64(a, s0_0, 2.0))
                R = lo_w - part
                if not s0_x > R:
                    continue
                t_0 = 2.0 * R / (s0_x - R)
                if not (1 << 12) <= t_0 <= (1 << 24) - 8:
                    continue
                for T in range(int(t_0) - 3, int(t_0) + 5):
                    if lo_w <= sum64([part, score64(T, s0_x, 2.0)]) < S_b:
                        case = _corpus(orc, np.array([cand[i], d]), np.array([s0_0, s0_x]), s1d, 1, k, n_docs, n_high,
                                       n_low, n_late, False, 0, rng, [t0, tx], [a, T], F_b, S_b, late_tf=(1, 2))
                        if case["tight_pruned"]:
                            return case
    raise AssertionError("no near-threshold fixture for a 2-term query")


def _find_a(orc, q, m, n_docs, lo_w, hi_w, rng, configs=300):
    """(df of term x, A's tfs over lanes 0 … m) with lo_w <= S_A < hi_w: A's coarse tfs on B's lanes at random, term x's
    df and tf solved for the rest."""
    for c in range(configs):
        # A holds some of B's lanes at tf 1 … 3: the rest R = lo_w − (their part) must be the score of one posting of a
        # term of df >= 300 (s0_x <= 3 ln(N / 300))
        coarse = [int(t) for t in rng.integers(1, 4, size=m)]
        for i in rng.permutation(m):
            if lo_w - sum64(score64(t, q.s0d[j], 2.0) for j, t in enumerate(coarse) if t) >= 8.0:
                break
            coarse[i] = 0
        part = sum64(score64(t, q.s0d[i], 2.0) for i, t in enumerate(coarse) if t)
        R = lo_w - part
        if not 8.0 <= R <= 3 * np.log(n_docs / 300):
            continue
        # s0_x in (R, R (1 + 2^-12)): tf_x = 2 R / (s0_x − R) >= 2^13
        dfx = np.arange(max(2, int((n_docs + 1) * np.exp(-R * (1 + 2.0 ** -12) / 3)) - 1),
                        int((n_docs + 1) * np.exp(-R / 3)) + 2)
        if len(dfx) == 0 or len(dfx) > 4096:
            continue
        s0x, _ = cache(orc, n_docs, dfx, 2.0, 0.0)
        for d, s0 in zip(dfx, s0x):
            if not s0 > R:
                continue
            t0 = 2.0 * R / (s0 - R)
            if t0 > (1 << 24) - 4:
                continue
            for tf in range(max(1, int(t0) - 3), int(t0) + 5):
                S = sum64([part, score64(tf, s0, 2.0)]) if part else float(score64(tf, s0, 2.0))
                if lo_w <= S < hi_w:
                    return int(d), coarse + [tf], float(s0)
    return None


def _with_a(orc, pick, cand, s0c, s1d, m, k, n_docs, n_high, n_low, n_late, dense, n_rare, rng, tf_b):
    q = Query(s0c[pick], s1d)
    F_b = float(q.filter_score(tf_b)[0])
    S_b = q.exact(tf_b)
    got = _find_a(orc, q, m, n_docs, _next_up(F_b), S_b, rng)
    if got is None:
        return None
    df_x, tf_a, s0_x = got
    return _corpus(orc, np.append(cand[pick], df_x), np.append(q.s0d, s0_x), s1d, m, k, n_docs, n_high, n_low, n_late,
                   dense, n_rare, rng, tf_b, tf_a, F_b, S_b)


def _corpus(orc, dfs, s0d, s1d, m, k, n_docs, n_high, n_low, n_late, dense, n_rare, rng, tf_b, tf_a, F_b, S_b,
            late_tf=(3, 3)):
    """The documents of near_threshold_case around B (tfs tf_b on lanes 0 … len(tf_b) − 1) and A (tf_a on lanes 0 … m)."""
    bl = len(tf_b)  # B's lanes: m, or m + 1 when B holds x as well
    qa = Query(s0d, s1d)
    S_a = qa.exact(tf_a)
    assert _next_up(F_b) <= S_a < S_b
    T = m + 1 + n_rare
    a_doc = n_high + (1 if n_rare else 0)
    low0 = a_doc + 1
    first = low0 + n_low
    b_doc = n_docs - 1
    lists = [([], []) for _ in range(T)]

    def put(doc, t, tf):
        lists[t][0].append(int(doc))
        lists[t][1].append(int(tf))

    for d in range(n_high):
        for t in range(bl):
            put(d, t, 30)
    for t in range(m + 1, T):
        put(n_high, t, 1)
    for t in range(m + 1):
        if tf_a[t]:
            put(a_doc, t, tf_a[t])
    for d in range(low0, first):
        put(d, 0, 1)
        put(d, 1, 1)
    used = np.array([len(lists[t][0]) + (n_late if t < 2 else 0) + (1 if t < bl else 0) for t in range(m + 1)])  # late, B
    region = int(min(dfs[:bl] - used[:bl])) - 8 if dense else 0
    extra = dfs - used - np.append(np.full(bl, region), np.zeros(m + 1 - bl, int))
    assert np.all(extra >= 0)
    singles = np.repeat(np.arange(m + 1), extra)
    rng.shuffle(singles)
    stop = b_doc - region
    late0 = (first + stop) // 2
    late = np.arange(late0, late0 + n_late)
    free = np.setdiff1d(np.arange(first, stop), late)
    stride = len(free) // (len(singles) + 1)
    assert stride >= 1
    docs = [(int(d), int(t), 1) for d, t in zip(free[np.arange(len(singles)) * stride], singles)]
    docs += [(int(d), t, late_tf[t]) for d in late for t in (0, 1)]
    for d, t, tf in sorted(docs):
        put(d, t, tf)
    S_late = float(score64(late_tf[0], qa.s0d[0], 2.0) + score64(late_tf[1], qa.s0d[1], 2.0))
    assert S_late < S_a
    for d in range(stop, b_doc):
        for t in range(bl):
            put(d, t, 1)
    for t in range(bl):
        put(b_doc, t, tf_b[t])
    post_off = np.zeros(T + 1, np.uint64)
    post_off[1:] = np.cumsum([len(d) for d, _ in lists])
    for t, (d, _) in enumerate(lists):
        assert np.all(np.diff(d) > 0) and (t > m or len(d) == dfs[t])
    post_doc = np.concatenate([np.asarray(d, np.uint32) for d, _ in lists])
    post_tf = np.concatenate([np.asarray(f, np.uint32) for _, f in lists])
    doc_len = np.maximum(np.bincount(post_doc, weights=post_tf, minlength=n_docs), 1).astype(np.uint32)
    # bounds (k_term_ub) and the pruned set at Sk = S_A over the m + 1 lanes of a single-pass query
    ubd = [float(max(score64(np.asarray(lists[t][1]), qa.s0d[t], 2.0))) * (1.0 + 2.0 ** -40) for t in range(m + 1)]
    pruned = pruned_lanes(ubd, S_a) if not n_rare else []
    tfb1 = list(tf_b) + [0] * (m + 1 - bl)
    F_probe = float(qa.filter_score(tfb1, order=probe_order(m + 1, pruned))[0])
    F_str = float(qa.filter_score(tfb1, order=[i for i in range(m + 1) if i not in pruned])[0]) if len(pruned) < bl else None
    Flo, _ = thresholds(S_a)
    Flo_p, FloT = thresholds(S_a, sum(ubd[i] for i in pruned))
    return dict(m=m, k=k, n_docs=n_docs, doc_len=doc_len, n_terms=T, post_off=post_off, post_doc=post_doc,
                post_tf=post_tf, query=np.arange(T, dtype=np.uint32), a_doc=a_doc, b_doc=b_doc, tf_a=tf_a, df=dfs,
                S_a=S_a, S_b=S_b, F_b=F_b, F_probe=F_probe, pruned=pruned, dense_from=stop, stride=stride,
                late=late, S_late=S_late, tf_b=list(tf_b), ubd=ubd,
                # kEps = 0 drops B, the shipped margin keeps it: without pruning (F_B against Flo), and with the terms
                # pruned at Sk = S_A (the streamed part against Flo − ub_ne, then the probe loop's Fres against FloT)
                tight=F_b < f32_rd(S_a), keeps=F_b >= Flo,
                tight_pruned=F_probe < f32_rd(S_a),
                keeps_pruned=F_probe >= FloT and (F_str is None or F_str >= Flo_p),
                max_keps=largest_rejecting_keps(F_b, S_a))


# The near-threshold cases of test_gpu_margins.py, one per kernel path the margin is load-bearing on.
# name: (near_threshold_case arguments, kernel path options, launches of the batch's one class)
MARGIN_CASES = {
    "plain_6_lanes": (dict(m=5, k=10, n_docs=1000000), KERNEL_PATHS["plain"], 1),    # class 8, KEEPW verification
    "class_16": (dict(m=15, k=10, n_docs=1000000), KERNEL_PATHS["plain"], 1),        # filter_term loop
    "class_32": (dict(m=31, k=10, n_docs=1000000), KERNEL_PATHS["plain"], 1),
    "seeded_4_lanes": (dict(m=3, k=10, n_docs=1000000), KERNEL_PATHS["seeded"], 2),  # seeded launch + (empty) hand-back launch
    "two_phase": (dict(m=3, k=10, n_docs=1000000), KERNEL_PATHS["twophase"], 2),     # suspend launch, resume launch (doc ids) finds B
    "two_pass": (dict(m=8, k=10, n_docs=1000000, n_rare=32), KERNEL_PATHS["plain"], 1),  # 41 lanes: B holds group 1 only
    "dense_window": (dict(m=4, k=10, n_docs=60000, binade=8.0, dense=True), KERNEL_PATHS["plain"], 1),
    "hbm_pool": (dict(m=3, k=1025, n_docs=1000000), KERNEL_PATHS["plain"], 1),       # k = 1025: pool in HBM, lazy cut
}


def hands_back(c, opts, prune):
    """The seeded launch's test at query start: a list of n_docs / seed_dense_div postings or more (dense), or with pruning
    on, a list of seed_prune_min or more that is 8 times the shortest (skewed)."""
    mx, mn = int(max(c["df"])), int(min(c["df"]))
    div = opts["seed_dense_div"]
    return bool((prune and mx >= opts["seed_prune_min"] and mx // 8 >= mn) or (div and mx >= c["n_docs"] // div + 1))
