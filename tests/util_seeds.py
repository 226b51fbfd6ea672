"""CPU restatement of how the seeded search kernel (k_search_ring, RING_SEEDED) hands its seeds to its doc windows, and
the corpora built to reach each branch of that hand-off on purpose.

  windows      util_prune.windows with a seeded launch's rings: 2^BM25X_DOCRING_LOG_R = 512 doc ids per run in the
               2..4-term classes, util_prune.alloc_rings("seeded8") per query in the 5..8-term class, a whole ring per run
               in the first round, no dense clamp; the last window ends at INF.
  list_seeds   the seed listing of one window (bm25x_search_ring.cuh, the seeds of a doc window): at k <= 32 (pool of 64,
               SST = 32) all M slices of 32 seed slots at once, above that slice by slice (min(k, 128) + 31) >> 5 slices per
               term, term-major, pausing for a verification pass whenever more than 64 entries are listed and slices
               remain (seeds_pending).  The list is empty when a window starts, so where listing pauses follows from the
               seed counts alone; the presence map's false alarms play no part.

Every corpus here uses b = 0 (util_prune.Lists): a posting's score depends on its term's df and its tf only, so which
postings are a term's champions, and in which order, is set by the tfs."""
import itertools
from types import SimpleNamespace

import numpy as np

import util_prune as up

INF = 0xFFFFFFFF
CHAMP_L = 128       # BM25X_CHAMP_L: champions per term, the seeded launch's largest limit
DOC_R = 512         # 2^BM25X_DOCRING_LOG_R: doc ids per run in the 2..4-term seeded classes
AL = 4              # doc ids per 16-byte TMA piece
LIST_FULL = 64      # the candidate list is verified once more than this many entries are listed
CLASSES = (2, 3, 4, 8)  # the seeded launch's term-count classes (5..8 live terms run in the 8-lane class)
MAX_WARPS = 20      # BM25X_RING_MAXWARPS: no class runs more warps per SM


def seeded_class(m):
    assert 2 <= m <= 8
    return m if m <= 4 else 8


def ring_sizes(dfs):
    """Doc ids per ring of each lane at query start."""
    M = seeded_class(len(dfs))
    return [DOC_R] * len(dfs) if M <= 4 else up.alloc_rings("seeded8", dfs).size


def seeds_of(c, t, k):
    """Term t's seeds at limit k: the doc ids of its first min(k, df, 128) champions, in champion order."""
    a, b = int(c.r.champ_off[t]), int(c.r.champ_off[t + 1])
    return c.r.champ.reshape(-1, 2)[a:b, 0][:min(k, CHAMP_L)].astype(np.int64)


def seeded_windows(c, lanes):
    """The windows of a seeded launch over the runs `lanes` (ascending term ids): [(lo, hi, rd after it)]."""
    R = ring_sizes([len(c.lists[t][0]) for t in lanes])
    return up.windows(c, lanes, 1, (), R=R, al=AL, n_chunks=None, first=None, clamp=False)


def list_seeds(seeds, M, k, lo, hi):
    """Seed listing in the window [lo, hi) of a class of M lanes (seeds: per live lane its seed doc ids).  Returns
    (listed, stops): listed = (lane, slot) in list order; stops = (next slice, "inside" | "between") where listing pauses
    because more than 64 entries are listed and slices remain: inside one term's slices, or between two terms."""
    m = len(seeds)
    inw = [np.flatnonzero((np.asarray(s) >= lo) & (np.asarray(s) < hi)) for s in seeds]
    if k <= 32:  # one slice per term, all M of them in one step (the list is empty when a window starts)
        return [(j, int(r)) for j in range(m) for r in inw[j]], []
    slices = (min(k, CHAMP_L) + 31) >> 5
    listed, stops, nc, ss = [], [], 0, 0
    while ss < M * slices:
        if nc > LIST_FULL:
            stops.append((ss, "inside" if ss % slices else "between"))
            nc = 0
        jj, s = divmod(ss, slices)
        ss += 1
        if jj >= m:
            continue
        new = [(jj, int(r)) for r in inw[jj] if 32 * s <= r < 32 * s + 32]
        listed += new
        nc += len(new)
    return listed, stops


def model(c, q, k):
    """Per window of query q at limit k: lo, hi, the seeds listed (lane, slot) and the listing stops."""
    lanes = sorted(int(t) for t in q)
    M = seeded_class(len(lanes))
    seeds = [seeds_of(c, t, k) for t in lanes]
    wins = []
    for lo, hi, _ in seeded_windows(c, lanes):
        listed, stops = list_seeds(seeds, M, k, lo, hi)
        wins.append(SimpleNamespace(lo=lo, hi=hi, listed=listed, stops=stops))
    return SimpleNamespace(lanes=lanes, M=M, seeds=seeds, windows=wins)


def check_model(mo, k):
    """The two properties every fixture must show: each seed is listed in exactly one window, and at k <= 32 no window
    lists more than 64 + 32·M seeds (the room the one-step listing relies on)."""
    listed = [e for w in mo.windows for e in w.listed]
    want = [(j, r) for j, s in enumerate(mo.seeds) for r in range(len(s))]
    assert len(listed) == len(set(listed)) and sorted(listed) == want, "a seed listed twice or never"
    if k <= 32:
        assert max(len(w.listed) for w in mo.windows) <= LIST_FULL + 32 * mo.M


def window_of(mo, lane, slot):
    return next(i for i, w in enumerate(mo.windows) if (lane, slot) in w.listed)


# ---- corpora ----

def _view(L):
    """What seeded_windows reads of a corpus under construction."""
    return SimpleNamespace(lists=[(np.array(sorted(d), np.int64),) for d in L.t])


def _disjoint(L, rng, terms, df, n_docs, exclude=()):
    """tf-1 postings until each term holds df, on documents no other of `terms` holds."""
    pool = np.setdiff1d(np.arange(n_docs), np.concatenate([np.fromiter(exclude, np.int64, len(exclude))] +
                                                          [np.fromiter(L.t[t], np.int64, len(L.t[t])) for t in terms]))
    pool = rng.permutation(pool)
    at = 0
    for t in terms:
        need = df - len(L.t[t])
        L.put(t, np.sort(pool[at:at + need]), 1)
        at += need


def _one_window(L, lanes, docs):
    """Index of the seeded window that holds all of `docs`, else None; and the number of windows."""
    wins = seeded_windows(_view(L), lanes)
    for i, (lo, hi, _) in enumerate(wins):
        if min(docs) >= lo and max(docs) < hi:
            return i, len(wins)
    return None, len(wins)


FULL_N = 200000
FULL_FILL = 3000
FULL_KS = (32, 31, 10, 1)


def full_slices_case(orc, shared, seed=0):
    """Per class, one query with as many live terms as the class has lanes.  Each term: 32 champions at tf 30 (the only
    postings above tf 1: its first 32 champions, equal scores across the query's terms), packed into a run of 32·M
    consecutive documents (document i of the run: term i mod M), and 3000 tf-1 postings on documents no other query
    term holds, spread over 200 000 documents so that a query has many windows.  The run starts at the first offset
    where one window of the model holds it all: every term lists a full slice of 32 seeds in that window (256 in one
    step in the 8-lane class).  shared: each champion document also holds the next term (tf 1), so every seed is the
    stream's business; else no other query term holds it and each seed enters alone."""
    rng = np.random.default_rng(4301 + shared)
    L = up.Lists(sum(CLASSES), FULL_N)
    qs, runs, t0 = [], [], 0
    for M in CLASSES:
        terms = list(range(t0, t0 + M))
        t0 += M
        for start in range(FULL_N // 3, FULL_N, 1013):
            run = start + np.arange(32 * M)
            for t in terms:
                L.t[t] = {}
            for i, d in enumerate(run.tolist()):
                L.put(terms[i % M], [d], 30)
                if shared:
                    L.put(terms[(i + 1) % M], [d], 1)
            _disjoint(L, rng, terms, FULL_FILL + len(L.t[terms[0]]), FULL_N, exclude=run.tolist())
            if _one_window(L, terms, run)[0] is not None:
                break
        else:
            raise AssertionError(f"no offset puts the champions of class {M} in one window")
        qs.append(terms)
        runs.append(run)
    c = L.build(orc)
    c.qs, c.runs, c.ks, c.shared = qs, runs, FULL_KS, shared
    return c


STOP_N = 100000
STOP_FILL = 1500
STOP_KS = (33, 64, 65, 96, 97, 127, 128)


def _stop_slots(M, k):
    """Which of each lane's first min(k, 128) seed slots sit in the window, so that its listing stops both inside a term's
    slices and between two terms: the fewest slots left out (the last d_s slots of slice s of lane 0), or all of them in
    when no choice makes both kinds of stop."""
    K = min(k, CHAMP_L)
    sizes = [min(32, K - 32 * s) for s in range((K + 31) >> 5)]
    cands = sorted(itertools.product(*[sorted({d for d in (0, 1, 2, 16, 31, 32) if d <= n}) for n in sizes]), key=sum)
    for d in cands:
        inw = [np.ones(K, bool) for _ in range(M)]
        for s_, ds in enumerate(d):
            inw[0][32 * s_ + sizes[s_] - ds:32 * s_ + sizes[s_]] = False
        _, stops = list_seeds([np.where(x, 0, 1) for x in inw], M, k, 0, 1)
        if {s for _, s in stops} == {"inside", "between"}:
            return inw
    return [np.ones(K, bool) for _ in range(M)]


def slice_stops_case(orc, seed=0):
    """Per class and per limit k of STOP_KS, one query with as many live terms as the class has lanes.  Every term has 128
    champions at distinct tfs (slot r: tf base + 127 - r; base 1000 for the last lane, whose champions outrank every
    other term's, 100 for the others) and 1500 tf-1 postings on documents of its own.  Of each lane's first min(k, 128)
    champions, those _stop_slots picks sit in one run of consecutive documents that one window of the model holds; the
    others and the champions past k lie before it, in other windows.  So that window lists more than 64 seeds
    before the last term's slices, and in each class at some k it stops both inside a term's slices and between two
    terms; the last term's seeds, the ones a missed slice would drop, are the query's top rows."""
    rng = np.random.default_rng(4401 + seed)
    groups = [(M, k) for M in CLASSES for k in STOP_KS]
    L = up.Lists(sum(M for M, _ in groups), STOP_N)
    qs, meta, t0 = [], [], 0
    for M, k in groups:
        terms = list(range(t0, t0 + M))
        t0 += M
        inm = _stop_slots(M, k)
        far = 2000 + np.arange(CHAMP_L * M)  # the champions outside the window: the first documents after 2000
        for start in range(STOP_N // 2, STOP_N, 1013):
            inw, out = [], []
            for t in terms:
                L.t[t] = {}
            for j, t in enumerate(terms):
                base = 1000 if j == M - 1 else 100
                for r in range(CHAMP_L):
                    here = r < len(inm[j]) and inm[j][r]
                    d = start + len(inw) if here else int(far[len(out)])
                    (inw if here else out).append(d)
                    L.put(t, [d], base + CHAMP_L - 1 - r)
            _disjoint(L, rng, terms, STOP_FILL + CHAMP_L, STOP_N, exclude=inw + out)
            w, _ = _one_window(L, terms, inw)
            if w is not None and (not out or _one_window(L, terms, inw + [max(out)])[0] is None):
                break
        else:
            raise AssertionError(f"no offset puts the champions of class {M}, k = {k} in one window")
        qs.append(terms)
        meta.append(SimpleNamespace(M=M, k=k, inm=inm, inw=inw))
    c = L.build(orc)
    c.qs, c.meta = qs, meta
    return c


EDGE_N = 100000
EDGE_KS = (1, 10, 32, 33, 128)


def edge_case(orc, seed=0):
    """Per class, one query with as many live terms as the class has lanes: lane 0 is term A, whose whole list lands in
    the first round (df <= its ring: it never bounds a window), the others bound the windows: 2500 postings each in the
    2..4-term classes; in the 8-lane class one run of 4500 (a ring of 1024) and six of 20, so that A's 500 postings get a
    ring of 512.  A's first champions sit in a
    middle window [lo, hi) that another run bounds: slot 0 on hi itself (the next window's), slot 1 on hi - 1, slot 2 on lo;
    slots 3 .. 9 in the last window (hi = INF), slot 3 on the last document, n_docs - 1.  Slot 0 has the highest tf of
    the query: listed in two windows, it would be two rows of the top 10."""
    rng = np.random.default_rng(4501 + seed)
    L = up.Lists(sum(CLASSES), EDGE_N)
    qs, meta, t0 = [], [], 0
    for M in CLASSES:
        terms = list(range(t0, t0 + M))
        t0 += M
        a, others = terms[0], terms[1:]
        df_a, df_o = (500, [4500] + [20] * 6) if M == 8 else (400, [2500] * (M - 1))
        for t, df in zip(others, df_o):
            L.put(t, np.sort(rng.choice(EDGE_N - 1, size=df, replace=False)), rng.integers(1, 4, size=df))
        R = ring_sizes([df_a] + df_o)
        assert R[0] >= df_a
        wins = up.windows(_view(L), others, 1, (), R=R[1:], al=AL, n_chunks=None, first=None, clamp=False)
        held = set().union(*(L.t[t] for t in others))
        w = next(i for i in range(len(wins) // 2, len(wins) - 1) if wins[i][1] - 1 > wins[i][0] and wins[i][1] - 1 not in held)
        lo, hi = wins[w][0], wins[w][1]
        last_lo = wins[-1][0]
        tail = [EDGE_N - 1] + sorted(rng.choice(np.arange(last_lo + 1, EDGE_N - 1), size=6, replace=False).tolist())
        champs = [hi, hi - 1, lo] + tail
        for r, d in enumerate(champs):
            L.put(a, [d], 60 - r)
        pool = np.setdiff1d(np.arange(EDGE_N), champs)
        L.put(a, np.sort(rng.choice(pool, size=df_a - len(champs), replace=False)), 1)
        qs.append(terms)
        meta.append(SimpleNamespace(M=M, w=w, lo=lo, hi=hi, champs=champs, df_a=df_a))
    c = L.build(orc)
    c.qs, c.meta = qs, meta
    return c


RESET_N = 50000
RESET_KS = (32, 33, 128)


def slot_reset_case(orc, seed=0):
    """48 "big" terms (df 200 .. 400: full champion lists, their first 128 postings at tf 50) and 48 "small" ones (df 3 ..
    20 at tf 1: fewer seeds than any limit of RESET_KS), all over the same 50 000 documents.  A seed slot left over
    from a big query would land in a window of the small query after it, with a score above all of its own rows."""
    rng = np.random.default_rng(4601 + seed)
    L = up.Lists(96, RESET_N)
    for t in range(48):
        df = int(rng.integers(200, 401))
        d = np.sort(rng.choice(RESET_N, size=df, replace=False))
        tf = np.ones(df, np.int64)
        tf[rng.choice(df, size=CHAMP_L, replace=False)] = 50
        L.put(t, d, tf)
    for t in range(48, 96):
        L.put(t, np.sort(rng.choice(RESET_N, size=int(rng.integers(3, 21)), replace=False)), 1)
    c = L.build(orc)
    c.big, c.small = np.arange(48), np.arange(48, 96)
    return c


def reset_queries(c, per_class, seed=0):
    """per_class queries per class, alternately of big and of small terms, as many live terms as the class has lanes."""
    rng = np.random.default_rng(4701 + seed)
    qs = []
    for M in CLASSES:
        for i in range(per_class):
            qs.append(sorted(rng.choice(c.big if i % 2 == 0 else c.small, size=M, replace=False).tolist()))
    return qs
