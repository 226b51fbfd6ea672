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


def near_threshold_case(orc, m, k, n_docs, *, binade=16.0, dense=False, n_rare=0, seed=0, tries=3000):
    """A corpus (b = 0, k1 = 2: exact regime) in which the margin kEps alone decides whether a top-k document survives.

    Query terms: ids 0 … m − 1 (B's terms), m (term x, A's knob) and, with n_rare, m + 1 … m + n_rare (df 1: the rarest,
    group 0 of a two-pass query).  Doc ids, in order: k − 1 − [n_rare > 0] "high" documents (B's terms, tf 30: above
    everything else); with n_rare, one document holding the rare terms; document A (term x at a large tf, a few of B's
    terms at tf <= 3, searched so that next_f32(F_B) <= S_A < S_B); 40 "low" documents (terms 0 and 1, tf 1); the fillers —
    single-term documents spread evenly (sparse) or, with `dense`, a block of documents holding every B term with tf 1 —
    with 40 "late low" documents (terms 0 and 1, tf 3: above every low document and filler, below S_A) halfway through
    them; and last, document B (B's m terms, tf 2).  The late low documents make the threshold S_A whatever order the
    early candidates were verified in: a kernel may cut the pool for the first time before the high documents or A are
    in it (the seeded kernel verifies its champion seeds and the documents of the lower runs first), and then, with
    nothing else above that first threshold, the k-th score would stay below S_A until B.  With them, the pool overflows
    again once A and the high documents are in, and is cut to exactly those k.  B's exact score beats S_A while B's f32
    filter score is below f32_rd(S_A): a kernel without the margin drops B.

    B's dfs are searched among the terms whose s0 (just above `binade`) rounds down most in f32, in the order that leaves
    F_B furthest below S_B."""
    rng = np.random.default_rng(seed)
    k1, b = 2.0, 0.0
    n_high = k - 1 - (1 if n_rare else 0)
    n_low = 40  # also the number of late low documents
    # s0 = 3 ln((N + 1) / (df + 0.5)) in [binade, 1.1 binade]
    cand = np.arange(int(n_docs * np.exp(-1.1 * binade / 3)) + 1, int(n_docs * np.exp(-binade / 3)))
    s0c, s1d = cache(orc, n_docs, cand, k1, b)
    assert np.all(s1d == 2.0) and len(cand) >= 2 * m
    rel = (s0c - s0c.astype(F32).astype(np.float64)) / s0c
    pool = np.argsort(-rel)[:max(60, 2 * m)]
    found = {}
    for _ in range(tries):
        pick = tuple(rng.choice(pool, size=m, replace=False))
        q = Query(s0c[list(pick)], s1d)
        F = float(q.filter_score([2] * m)[0])
        S = q.exact([2] * m)
        if S > _next_up(F):
            found[pick] = (S - _next_up(F)) / S
    for pick in sorted(found, key=lambda p: -found[p])[:40]:
        case = _with_a(orc, np.array(pick), cand, s0c, s1d, m, k, n_docs, n_high, n_low, dense, n_rare, rng)
        if case is not None and (case["tight_pruned"] or m + 1 > 8 or n_rare):
            return case
    raise AssertionError(f"no near-threshold fixture for m={m}")


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


def _with_a(orc, pick, cand, s0c, s1d, m, k, n_docs, n_high, n_low, dense, n_rare, rng):
    q = Query(s0c[pick], s1d)
    tf_b = [2] * m
    F_b = float(q.filter_score(tf_b)[0])
    S_b = q.exact(tf_b)
    got = _find_a(orc, q, m, n_docs, _next_up(F_b), S_b, rng)
    if got is None:
        return None
    df_x, tf_a, s0_x = got
    qa = Query(np.append(q.s0d, s0_x), s1d)
    S_a = qa.exact(tf_a)
    assert _next_up(F_b) <= S_a < S_b
    dfs = np.append(cand[pick], df_x)
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
        for t in range(m):
            put(d, t, 30)
    for t in range(m + 1, T):
        put(n_high, t, 1)
    for t in range(m + 1):
        if tf_a[t]:
            put(a_doc, t, tf_a[t])
    for d in range(low0, first):
        put(d, 0, 1)
        put(d, 1, 1)
    used = np.array([len(lists[t][0]) + (n_low if t < 2 else 0) + (1 if t < m else 0) for t in range(m + 1)])  # late, B
    region = int(min(dfs[:m] - used[:m])) - 8 if dense else 0
    extra = dfs - used - np.append(np.full(m, region), 0)
    assert np.all(extra >= 0)
    singles = np.repeat(np.arange(m + 1), extra)
    rng.shuffle(singles)
    stop = b_doc - region
    late0 = (first + stop) // 2
    late = np.arange(late0, late0 + n_low)
    free = np.setdiff1d(np.arange(first, stop), late)
    stride = len(free) // (len(singles) + 1)
    assert stride >= 1
    docs = [(int(d), int(t), 1) for d, t in zip(free[np.arange(len(singles)) * stride], singles)]
    docs += [(int(d), t, 3) for d in late for t in (0, 1)]
    for d, t, tf in sorted(docs):
        put(d, t, tf)
    S_late = float(score64(3, qa.s0d[0], 2.0) + score64(3, qa.s0d[1], 2.0))
    assert S_late < S_a
    for d in range(stop, b_doc):
        for t in range(m):
            put(d, t, 1)
    for t in range(m):
        put(b_doc, t, 2)
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
    tfb1 = tf_b + [0]
    F_probe = float(qa.filter_score(tfb1, order=probe_order(m + 1, pruned))[0])
    F_str = float(qa.filter_score(tfb1, order=[i for i in range(m + 1) if i not in pruned])[0]) if len(pruned) < m else None
    Flo, _ = thresholds(S_a)
    Flo_p, FloT = thresholds(S_a, sum(ubd[i] for i in pruned))
    return dict(m=m, k=k, n_docs=n_docs, doc_len=doc_len, n_terms=T, post_off=post_off, post_doc=post_doc,
                post_tf=post_tf, query=np.arange(T, dtype=np.uint32), a_doc=a_doc, b_doc=b_doc, tf_a=tf_a, df=dfs,
                S_a=S_a, S_b=S_b, F_b=F_b, F_probe=F_probe, pruned=pruned, dense_from=stop, stride=stride,
                late=late, S_late=S_late,
                # kEps = 0 drops B, the shipped margin keeps it: without pruning (F_B against Flo), and with the terms
                # pruned at Sk = S_A (the streamed part against Flo − ub_ne, then the probe loop's Fres against FloT)
                tight=F_b < f32_rd(S_a), keeps=F_b >= Flo,
                tight_pruned=F_probe < f32_rd(S_a),
                keeps_pruned=F_probe >= FloT and (F_str is None or F_str >= Flo_p),
                max_keps=largest_rejecting_keps(F_b, S_a))
