"""CPU model of what the `allow` bitmap of bm25x_search_batch changes in k_search_ring (bm25x_search_ring.cuh), and the
corpora built to put a bitmap against each decision on purpose.

The kernel tests the bitmap after the f32 filter and before pool_insert (the verification pass, and the seeded
kernel's hit-list flush), so the pool only ever holds allowed documents: every threshold the kernel derives from it (the
k-th score Sk, the single-posting limit wlim, MaxScore's prune set, the two-phase hand-over) is at most the k-th score of
the allowed documents, and a batch with a bitmap never reaches the seeded kernel (seeded_class), whose seeds are each
term's first min(k, 128) champions whether or not the bitmap allows them.

  bitmap        the bitmap of a set of documents (bit d of byte d >> 3), padding bits past n_docs optional.
  topk          the filtered top-k (score desc, doc asc) from the exact f64 scores.
  beyond_seeds  documents of a filtered top-k that hold one query term and are not among its seeds: a seeded launch
                would never list them.
  prune_band    the prune set at the second chunk boundary of a prune_case under a bitmap (util_prune.band on the allowed
                documents of the first window), or that no threshold the allowed documents give can prune at all.
  handover      the two-phase launch's suspend test at every chunk boundary, bracketed by the least and the most the
                threshold can be there (handover_before: the same test for a near-threshold case, whose threshold is S_A).
  dense_window  the plain kernel's window holding given documents, and whether its postings take the dense accumulator.
  growing       growing documents whose decisive ones a bitmap partly clears, and the bitmap the reference sees when
                allow_growing is cut at allow_growing_docs.

Every corpus here uses b = 0 (util_prune.Lists): a posting's score depends on its term's df and its tf only."""
from types import SimpleNamespace

import numpy as np

import util_filter as uf
import util_prune as up
import util_seeds as us


def bitmap(n_docs, allowed=None, cleared=(), pad=False):
    """Bitmap of the documents `allowed` (default all) minus `cleared`.  pad: the bits past n_docs in the last byte set."""
    ok = np.zeros(n_docs, bool)
    if allowed is None:
        ok[:] = True
    else:
        ok[np.asarray(allowed, np.int64)] = True
    ok[np.asarray(list(cleared), np.int64)] = False
    nb = (n_docs + 7) // 8
    bits = np.zeros(nb * 8, bool)
    bits[:n_docs] = ok
    if pad:
        bits[n_docs:] = True
    return np.packbits(bits, bitorder="little")


def allowed_mask(allow, n_docs):
    return np.unpackbits(np.asarray(allow, np.uint8), bitorder="little")[:n_docs].astype(bool)


def matches(c, q):
    """Documents holding at least one term of q, ascending."""
    return np.unique(np.concatenate([c.lists[int(t)][0] for t in q])).astype(np.int64)


def topk(c, q, k, allow=None):
    """(docs, scores) of the filtered top-k in the canonical order (score desc, doc asc)."""
    s = up.doc_scores(c, q)
    cand = matches(c, q)
    if allow is not None:
        cand = cand[allowed_mask(allow, c.n_docs)[cand]]
    order = np.lexsort((cand, -s[cand]))[:k]
    return cand[order], s[cand[order]]


def holders(c, q, d):
    return [int(t) for t in q if d in c.sets[int(t)]]


def beyond_seeds(c, q, k, allow):
    """Documents of the filtered top-k that hold exactly one query term and are not among that term's seeds at limit k
    (util_seeds.seeds_of: its first min(k, df, 128) champions)."""
    docs, _ = topk(c, q, k, allow)
    seeds = {int(t): set(us.seeds_of(c, int(t), k).tolist()) for t in q}
    out = []
    for d in docs.tolist():
        h = holders(c, q, d)
        if len(h) == 1 and d not in seeds[h[0]]:
            out.append(d)
    return out


def with_sets(c):
    c.sets = [set(d.tolist()) for d, _ in c.lists]
    return c


# ---- filtered champions ----

CHAMP_N = 100003         # n_docs % 8 != 0: the all-ones bitmap has padding bits
CHAMP_RANKED = 300       # postings per term at distinct tfs (400 - r): champion r of the term is its r-th of them
CHAMP_KS = (1, 10, 32, 33, 128, 129, 224)
CHAMP_KINDS = ("one", "every", "all_but_last", "past_cut")


def champion_case(orc, seed=0):
    """Per seeded class (2, 3, 4, 8 live terms) one query.  Every term holds 300 ranked postings (tf 400 - r) and tf-1
    postings after them, each on a document no other term of its query holds; lane 0 (df 1000) outscores the other lanes
    (df 3000) at every rank, so the filtered top k is made of lane 0's best allowed postings."""
    rng = np.random.default_rng(4801 + seed)
    n_terms = sum(us.CLASSES)
    L = up.Lists(n_terms, CHAMP_N)
    free = rng.permutation(CHAMP_N)
    ranked_all, at, qs = [], 0, []
    for M in us.CLASSES:
        q = list(range(sum(us.CLASSES[:us.CLASSES.index(M)]), sum(us.CLASSES[:us.CLASSES.index(M)]) + M))
        for t in q:
            docs = free[at:at + CHAMP_RANKED]
            at += CHAMP_RANKED
            L.put(t, docs, 400 - np.arange(CHAMP_RANKED))
            ranked_all.append(docs)
        qs.append(q)
    ranked = set(np.concatenate(ranked_all).tolist())
    for q in qs:
        us._disjoint(L, rng, q[:1], 1000, CHAMP_N, exclude=ranked)
        us._disjoint(L, rng, q[1:], 3000, CHAMP_N, exclude=ranked | set(L.t[q[0]]))
    c = with_sets(L.build(orc))
    c.qs = qs
    return c


def champion_bitmap(c, kind, k):
    """The bitmap of one kind over every query of champion_case at limit k."""
    clear, allow = set(), None
    for q in c.qs:
        for j, t in enumerate(q):
            seeds = us.seeds_of(c, t, k).tolist()
            if kind == "one" and j == 0 or kind == "every":
                clear |= set(seeds)
            elif kind == "all_but_last":
                clear |= set(seeds[:-1])
    if kind == "past_cut":  # only the postings ranked right after the 128-entry champion lists
        ch = c.r.champ.reshape(-1, 2)[:, 0]
        allow = []
        for q in c.qs:
            for t in q:
                d, tf = c.lists[t]
                allow += d[(tf <= 400 - us.CHAMP_L) & (tf > 400 - CHAMP_RANKED)].tolist()
        assert not set(allow) & set(ch.tolist())
    return bitmap(c.n_docs, allow, clear)


# ---- unfilled pools ----

POOL_N = 100000
POOL_KS = (1, 10, 32, 33, 224, 225, 1024, 1025, 65535)


def pool_case(orc, seed=0):
    """A 3-term query (class 4) and an 8-term one over 100 000 documents, with about 78 000 and 75 000 or more matches:
    enough for a bitmap of k + 1 allowed matches at the largest limit."""
    rng = np.random.default_rng(4901 + seed)
    L = up.Lists(11, POOL_N)
    for t in range(3):
        L.put(t, np.sort(rng.choice(POOL_N, size=40000, replace=False)), rng.integers(1, 8, size=40000))
    for t in range(3, 11):
        df = int(rng.integers(15000, 30000))
        L.put(t, np.sort(rng.choice(POOL_N, size=df, replace=False)), rng.integers(1, 8, size=df))
    c = with_sets(L.build(orc))
    c.qs = [[0, 1, 2], list(range(3, 11))]
    return c


def pool_bitmap(c, q, k, n_allowed, seed=0):
    """n_allowed matches of query q allowed (a random choice), nothing else; q runs alone in its batch."""
    rng = np.random.default_rng(5001 + 7 * k + n_allowed + seed)
    mt = matches(c, q)
    assert len(mt) >= n_allowed
    return bitmap(c.n_docs, rng.choice(mt, size=n_allowed, replace=False))


LAST_KS = (1, 10, 32, 33)  # the last window of pool_case's 3-term query holds some 80 matches


def last_window_bitmap(c, q, k):
    """The first k + 1 matches of query q in the last window allowed, nothing else."""
    lo = last_window(c, q)
    mt = matches(c, q)
    return bitmap(c.n_docs, mt[mt >= lo][:k + 1])


def last_window(c, q):
    """lo of the plain kernel's last window (hi = INF) for query q: util_prune.windows with the 2..4-term class's rings."""
    return up.windows(c, sorted(q), 99, [], n_chunks=None)[-1][0]


# ---- two-phase hand-over ----

TWO_N = 100000
TWO_DF = 20000
TWO_REGION = 400  # documents per region: more than the largest pool KP = 256, so a cut inside it holds k of them
TWO_E0, TWO_L0 = 2000, 30000
TWO_KS = (1, 10, 32, 33, 128, 129, 224)
TWO_KINDS = ("before", "after", "short", "low")


def two_phase_case(orc, seed=0):
    """Per class of the two-phase launches (2, 3, 4 live terms) one query of equal dfs (20 000).  Region E (400 documents
    from 2000 on, every third one) holds every query term at tf 30, region L (400 from 30 000 on) every one at tf 40: each
    region document outscores any single posting, an L document any E one.  Every other posting has tf 1 and lies on a
    document no other term of its query holds, so no document outside E and L scores above one posting."""
    rng = np.random.default_rng(5101 + seed)
    E = TWO_E0 + 3 * np.arange(TWO_REGION)
    Lr = TWO_L0 + 3 * np.arange(TWO_REGION)
    L = up.Lists(9, TWO_N)
    qs, t0 = [], 0
    for M in (2, 3, 4):
        q = list(range(t0, t0 + M))
        t0 += M
        for t in q:
            L.put(t, E, 30)
            L.put(t, Lr, 40)
        us._disjoint(L, rng, q, TWO_DF, TWO_N, exclude=set(E.tolist()) | set(Lr.tolist()))
        qs.append(q)
    c = with_sets(L.build(orc))
    c.qs, c.E, c.L = qs, E, Lr
    return c


def two_phase_bitmap(c, kind, k, seed=0):
    """before: every other document of L cleared, from L's first one on (E sets a threshold no single posting reaches,
    and L, allowed and cleared documents alike, comes after it: the resume launch meets the bitmap).  after: E cleared
    (the threshold reaches that level only in L).  short: k - 1 allowed matches per query (the pool never fills).  low:
    E and L cleared (no threshold ever rises above a single posting)."""
    if kind == "before":
        return bitmap(c.n_docs, cleared=c.L[0::2].tolist())
    if kind == "after":
        return bitmap(c.n_docs, cleared=c.E.tolist())
    if kind == "low":
        return bitmap(c.n_docs, cleared=c.E.tolist() + c.L.tolist())
    rng = np.random.default_rng(5201 + k + seed)
    allow = []
    for q in c.qs:  # documents no other query's term holds: each query sees exactly its own k - 1
        own = np.setdiff1d(matches(c, q), np.concatenate([matches(c, o) for o in c.qs if o is not q]))
        allow += rng.choice(own, size=k - 1, replace=False).tolist()
    return bitmap(c.n_docs, allow)


def _kth(scores_desc, k):
    return float(scores_desc[k - 1]) if len(scores_desc) >= k else None


def handover(c, q, k, allow, prune):
    """The suspend test of RING_SUSPEND at every chunk boundary of query q (2..4 terms, pruning on or off): it suspends
    once a threshold exists, no streamed run's bound reaches Flo (wlim saturated) and at least BM25X_SUSPEND_MIN postings
    of the streamed runs are left.  The threshold at a boundary is bracketed: at most the k-th score of the allowed
    documents consumed so far (the pool holds allowed documents only), at least their KP-th (a cut keeps the top k of
    everything inserted; fewer than KP entries can have been inserted since the last one).  Returns (first boundary where
    the test can pass, first where it must, windows); a boundary j is the one after chunk j (1-based), whose documents
    below win[j - 1][1] have all been consumed.  The windows are those without pruning: the model asserts that no
    boundary before the hand-over prunes."""
    lanes = sorted(int(t) for t in q)
    win = up.windows(c, lanes, 99, [], n_chunks=None)
    s = up.doc_scores(c, lanes)
    ok = allowed_mask(allow, c.n_docs)
    mt = matches(c, lanes)
    mt = mt[ok[mt]]
    kp = uf.pool_capacity(k)
    ubd = [float(c.r.ubd[t]) for t in lanes]

    def passes(Sk, rd):
        if Sk is None:
            return False
        P = up.prune_at(c, lanes, Sk) if prune else []
        flo = Sk * (1.0 - uf.KEPS) - sum(ubd[i] for i in P)
        act = [i for i in range(len(lanes)) if i not in P]
        return all(ubd[i] < flo for i in act) and sum(int(c.df[lanes[i]]) - rd[i] for i in act) >= up.SUSPEND_MIN

    can = must = None
    for j, (_, hi, rd) in enumerate(win, start=1):
        if hi == us.INF:
            break
        done = np.sort(s[mt[mt < hi]])[::-1]
        Sk_hi = _kth(done, k)
        if can is None:
            if passes(Sk_hi, rd):
                can = j
            elif prune:  # nothing pruned before the hand-over: the windows are the unpruned ones
                assert Sk_hi is None or up.prune_at(c, lanes, Sk_hi) == [], (j, Sk_hi)
        if passes(_kth(done, kp), rd):
            must = j
            break
    return can, must, win


# ---- pruning ----

def prune_bitmaps(c, kp, seed=0):
    """Two bitmaps of a prune_case: `band` keeps the band (the first window's documents) and clears half of the other
    documents at random; `cleared` clears the band and every document that scores at least twice the lowest bound of
    the query's terms, so that no threshold the allowed documents give reaches the prune rule (ALPHA = 1/2)."""
    rng = np.random.default_rng(5301 + seed)
    lanes = [int(t) for t in c.q]
    s = up.doc_scores(c, c.q)
    mt = matches(c, c.q)
    band = np.arange(c.band_docs)
    rest = np.setdiff1d(mt, band)
    keep = bitmap(c.n_docs, cleared=rng.choice(rest, size=len(rest) // 2, replace=False).tolist())
    low = 2.0 * min(float(c.r.ubd[t]) for t in lanes)
    clear = bitmap(c.n_docs, cleared=sorted(set(band.tolist()) | set(mt[s[mt] >= low].tolist())))
    return dict(band=keep, cleared=clear)


def prune_band(c, k, kp, allow):
    """(prune set at the second boundary at both ends of the band of the allowed first-window documents, or None when
    they do not cut the pool; prune set at the k-th allowed score, the highest threshold the kernel can reach)."""
    lanes = [int(t) for t in c.q]
    _, docs = up.first_window(c, lanes)
    docs = docs[allowed_mask(allow, c.n_docs)[docs]]
    top, _ = topk(c, c.q, k, allow)
    s = up.doc_scores(c, c.q)
    final = up.prune_at(c, lanes, float(s[top[-1]])) if len(top) == k else []
    if len(docs) < uf.cut_trigger(k, kp, False):
        return None, final
    w = np.sort(s[docs])[::-1]
    P_lo, P_hi = up.prune_at(c, lanes, float(w[-1])), up.prune_at(c, lanes, float(w[k - 1]))
    assert P_lo == P_hi, (P_lo, P_hi)
    return P_lo, final


# roles of util_prune.prune_case (lanes in ascending term id): one head of bound 0.22 pruned at the band in each class
# that splits its rings per query, the other terms never pruned (H_HIGH: bound 6.3 > B / 2, F: 8.5)
_S, _F, _H_LOW, _H_HIGH = ("S",), ("F",), ("H", 80000, 1), ("H", 5000, 30)
PRUNE_ROLES = {
    "class8": [_S, _H_HIGH, _H_LOW, _S, _H_HIGH, _H_HIGH],
    "class16": [_S, _S, _H_HIGH, _H_HIGH, _H_LOW, _H_HIGH, _H_HIGH, _H_HIGH, _H_HIGH],
    "class32": [_S, _S, _H_HIGH, _H_LOW, _H_HIGH] + [_F] * 13,
}
PRUNE_K, PRUNE_KP = 10, 64


def prune_fixture(orc, name):
    c = with_sets(up.prune_case(orc, PRUNE_ROLES[name], PRUNE_K))
    c.head = PRUNE_ROLES[name].index(_H_LOW)
    return c


# ---- margin ----

# near_threshold_case arguments (built at k = 10) and the path the case is run on, at k = 1 with the high documents
# cleared: the plain 8-term class (6 lanes) and the two-phase class of 4 lanes (with pruning off B is scored by the
# resume launch; with pruning on the query stays in the suspend launch, see handover_before)
MARGIN = {"plain8": (dict(m=5, k=10, n_docs=1000000), "plain"),
          "two_phase": (dict(m=3, k=10, n_docs=1000000), "twophase")}


def margin_case(orc, name):
    return uf.near_threshold_case(orc, **MARGIN[name][0])


def margin_bitmap(c):
    """The k - 1 high documents (ids 0 .. a_doc - 1) cleared: A is the best allowed document before B."""
    return bitmap(c["n_docs"], cleared=range(c["a_doc"]))


def handover_before(c, k, allow, prune, upto):
    """The hand-over of a near_threshold_case (a dict) at limit k under `allow`, with the threshold S_A: the first window
    boundary after the documents up to `upto` (A and the low documents after it: the pool is cut with A as its best
    allowed entry there) at which every streamed term's bound is below Flo and at least BM25X_SUSPEND_MIN postings are
    left.  Returns that boundary's hi (None: no hand-over).  Windows without pruning; the pruned set of the case at S_A
    when `prune`."""
    T = c["n_terms"]
    off = c["post_off"].astype(np.int64)
    lists = [(c["post_doc"][off[t]:off[t + 1]].astype(np.int64),) for t in range(T)]
    view = SimpleNamespace(lists=lists)
    lanes = list(range(T))
    P = c["pruned"] if prune else []
    flo = c["S_a"] * (1.0 - uf.KEPS) - sum(c["ubd"][i] for i in P)
    act = [i for i in lanes if i not in P]
    if not all(c["ubd"][i] < flo for i in act):
        return None
    for lo, hi, rd in up.windows(view, lanes, 99, [], n_chunks=None):
        if hi == us.INF:
            return None
        if hi > upto and sum(len(lists[i][0]) - rd[i] for i in act) >= up.SUSPEND_MIN:
            return hi
    return None


# ---- dense window ----

DENSE_N = 60000
DENSE_KS = (10, 32, 33)
DENSE_BEST = 20
DENSE_ACC = 512  # ACC_DOCS of the 2..4-term plain classes: 2^11 map bytes / 4
DENSE_T = 48     # BM25X_RING_DENSE_T


def dense_case(orc, seed=0):
    """A 3-term query whose lists each hold a random half of 60 000 documents at tf 1, so that most windows of the plain
    kernel are dense and clamped to its 512-document accumulator.  In one clamped window in the middle, 20 documents that
    hold all three terms get tf 30 (the best of the query: `best`); in another, 20 get tf 20 (`next`).  Only tfs change,
    so the windows are those of the tf-1 lists."""
    rng = np.random.default_rng(5401 + seed)
    L = up.Lists(3, DENSE_N)
    for t in range(3):
        L.put(t, np.sort(rng.choice(DENSE_N, size=DENSE_N // 2, replace=False)), 1)
    view = SimpleNamespace(lists=[(np.array(sorted(d), np.int64),) for d in L.t])
    win = up.windows(view, [0, 1, 2], 99, [], n_chunks=None)
    clamped = [w for w in win[2:-1] if w[1] - w[0] == DENSE_ACC]
    all3 = sorted(set(L.t[0]) & set(L.t[1]) & set(L.t[2]))
    picks = []
    for lo, hi, _ in (clamped[len(clamped) // 2], clamped[len(clamped) // 4]):
        inw = [d for d in all3 if lo <= d < hi]
        picks.append(sorted(rng.choice(inw, size=DENSE_BEST, replace=False).tolist()))
    for t in range(3):
        L.put(t, picks[0], 30)
        L.put(t, picks[1], 20)
    c = with_sets(L.build(orc))
    c.q, c.best, c.next, c.win = [0, 1, 2], picks[0], picks[1], win
    return c


def dense_window(c, docs):
    """(lo, hi, dense) of the plain kernel's window holding all of `docs`: dense is the kernel's test on the postings the
    window consumes (Σn² − Σn²ᵢ > 2 · BM25X_RING_DENSE_T · span)."""
    for j, (lo, hi, rd) in enumerate(c.win):
        if lo <= min(docs) and max(docs) < hi:
            prev = c.win[j - 1][2] if j else [0] * len(rd)
            n = [a - b for a, b in zip(rd, prev)]
            return lo, hi, sum(n) ** 2 - sum(x * x for x in n) > 2 * DENSE_T * (hi - lo)
    return None


# ---- growing segment ----

GROW_N = 3000          # growing documents
GROW_CUT = 2600        # allow_growing_docs: the bitmap covers ordinals below it only
GROW_KS = (10, 128, 224)


def growing_docs(c, seed=0):
    """Growing documents over the two-phase queries' terms: per query 120 documents holding every term of it at tf 50
    (above every sealed document: `decisive`, spread over all ordinals, some past GROW_CUT), the rest one random term at
    tf 1.  Returns (elem_off, elem_term, elem_tf, doc_len, decisive ordinals)."""
    rng = np.random.default_rng(5501 + seed)
    terms = [t for q in c.qs for t in q]
    owner = np.full(GROW_N, -1)
    dec = rng.choice(GROW_N, size=120 * len(c.qs), replace=False)
    for i, q in enumerate(c.qs):
        owner[dec[120 * i:120 * (i + 1)]] = i
    off, et, ef = [0], [], []
    for g in range(GROW_N):
        if owner[g] >= 0:
            q = c.qs[owner[g]]
            et += q
            ef += [50] * len(q)
        else:
            et.append(int(rng.choice(terms)))
            ef.append(1)
        off.append(len(et))
    tf = np.array(ef, np.uint32)
    doc_len = np.add.reduceat(tf, np.array(off[:-1])).astype(np.uint32)
    return (np.array(off, np.uint64), np.array(et, np.uint32), tf, doc_len, np.sort(dec))


def growing_bitmap(dec):
    """allow_growing: every other decisive document below GROW_CUT cleared; every bit from GROW_CUT on set (the cut
    must drop those documents)."""
    return bitmap(GROW_N, cleared=dec[dec < GROW_CUT][0::2].tolist()), GROW_CUT


def growing_reference_bitmap(allow_g, cut):
    """The bitmap the reference sees: allow_growing's bits below the cut."""
    ok = allowed_mask(allow_g, GROW_N)
    ok[cut:] = False
    return bitmap(GROW_N, np.flatnonzero(ok))
