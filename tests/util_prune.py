"""CPU restatement of what k_search_ring (bm25x_search_ring.cuh) decides at run time around MaxScore pruning, and the
corpora built to reach those decisions on purpose.

  alloc_rings    the per-query split of a warp's ring budget in the classes of 8 or more terms (RCfg::ADAPT): a power of
                 two per streamed run, in proportion to df, with the branch each run took.
  first_window   the doc window of the first chunk: every run loads BM25X_RING_INIT postings, and the runs with postings
                 left in HBM bound the window by their last landed document.
  windows        the windows of the first chunks (or of all of them) of a class of at most 8 terms, plain or seeded.
  pruned_lanes   the prune rule at a chunk boundary (util_filter.pruned_lanes, with ub_oth of a two-pass query's pass 0).

Every corpus here uses b = 0 (the fieldnorm drops out of the score): a posting's score depends on its term's df and its
tf only, so score bands and bit-equal bounds are built from tfs and dfs alone.  The exact numbers still come from the
restatement of the index arrays (util_index.restate: ubd, blk_ub, per-posting f64 scores)."""
from types import SimpleNamespace

import numpy as np

import util_filter as uf
from util_index import restate

INIT = 32            # BM25X_RING_INIT: postings per run in the first load
SUSPEND_MIN = 4096   # BM25X_SUSPEND_MIN
BLOCK = 128          # BM25X_BLOCK
K1, B = 1.2, 0.0

# the four instantiations that size their rings per query: (M, R, budget, LOG_R, LOG_RMAX, AL)
RING_CLASSES = {
    "plain8": (8, 256, 2048, 8, 10, 2),
    "plain16": (16, 128, 2048, 7, 9, 2),
    "plain32": (32, 128, 4096, 7, 9, 2),
    "seeded8": (8, 512, 4096, 9, 10, 4),   # doc-id rings (RCfg::DOCRING): 4 postings per 16 bytes
}
LOG_RMIN = 6
BRANCHES = ("near", "down", "clamp", "halve", "halve2", "double")


def alloc_rings(cls, dfs, streamed=None):
    """alloc_rings of k_search_ring for lanes 0 .. len(dfs) - 1 (streamed: the lanes still streamed, default all).
    Returns sizes / bases / rlog per lane (0 for a lane that is not streamed), small (every ring <= 2^LOG_R) and the
    branches taken: near / down (rounded to the nearest power of two, or down because the nearest ones did not fit),
    clamp (a ring lowered to the smallest power of two >= the padded list), halve (overshoot halvings, a count) and
    double (rounds of the doubling loop, a count)."""
    M, R, BUDGET, LOG_R, LOG_RMAX, AL = RING_CLASSES[cls]
    m = len(dfs)
    assert m <= M
    streamed = set(range(m)) if streamed is None else set(streamed)
    mine = [i in streamed for i in range(m)]
    sumdf = sum(int(dfs[i]) for i in range(m) if mine[i])
    dfpad = [(int(d) + AL - 1) & ~(AL - 1) for d in dfs]
    lo2, near2, clamp_lo, clamp_near = [0] * m, [0] * m, [False] * m, [False] * m
    for i in range(m):
        if not mine[i]:
            continue
        share = (BUDGET * int(dfs[i])) // sumdf
        l2 = share.bit_length() - 1 if share > 1 else 0
        n2 = l2 + (1 if share * share >= (2 << (2 * l2)) else 0)
        l2 = min(max(l2, LOG_RMIN), LOG_RMAX)
        n2 = min(max(n2, LOG_RMIN), LOG_RMAX)
        while l2 > LOG_RMIN and (1 << (l2 - 1)) >= dfpad[i]:
            l2 -= 1
            clamp_lo[i] = True
        while n2 > LOG_RMIN and (1 << (n2 - 1)) >= dfpad[i]:
            n2 -= 1
            clamp_near[i] = True
        lo2[i], near2[i] = l2, n2
    fits = sum(1 << near2[i] for i in range(m) if mine[i]) <= BUDGET
    br = dict(near=0, down=0, clamp=0, halve=0, halve2=0, double=0)
    rlog = [0] * m
    size = [0] * m
    for i in range(m):
        if mine[i]:
            rlog[i] = near2[i] if fits else lo2[i]
            size[i] = 1 << rlog[i]
            br["clamp"] += int(clamp_near[i] if fits else clamp_lo[i])
    br["near" if fits else "down"] = 1
    used = sum(size)
    while used > BUDGET:
        big = max(size)
        who = size.index(big)  # the lowest lane of the largest rings
        rlog[who] -= 1
        size[who] >>= 1
        used -= big >> 1
        br["halve"] += 1
    br["halve2"] = int(br["halve"] >= 2)
    while True:
        can = [mine[i] and rlog[i] < LOG_RMAX and size[i] < dfpad[i] for i in range(m)]
        extra = sum(size[i] for i in range(m) if can[i])
        if extra == 0 or used + extra > BUDGET:
            break
        for i in range(m):
            if can[i]:
                rlog[i] += 1
                size[i] <<= 1
        used += extra
        br["double"] += 1
    bases = list(np.cumsum([0] + size[:-1]))
    return SimpleNamespace(size=size, base=[int(b) for b in bases], rlog=rlog, used=used, budget=BUDGET,
                           small=max(rlog) <= LOG_R, branches=br)


def moved(before, after, streamed):
    """Streamed lanes whose ring changed place or size between two geometries."""
    return [i for i in streamed if (before.base[i], before.size[i]) != (after.base[i], after.size[i])]


def pass_lanes(q_terms, df):
    """The lanes of each pass: one group in ascending term id, or for 33 .. 64 terms the 32 rarest (by df, then id)
    first and the others after them (bm25x_canonicalise)."""
    q = sorted(int(t) for t in q_terms)
    if len(q) <= 32:
        return [q]
    g0 = sorted(sorted(q, key=lambda t: (int(df[t]), t))[:32])
    return [g0, sorted(set(q) - set(g0))]


def ring_class(n, seeded=False):
    if seeded:
        assert 5 <= n <= 8
        return "seeded8"
    return "plain8" if n <= 8 else "plain16" if n <= 16 else "plain32"


def query_geometries(q_terms, df, seeded=False):
    """alloc_rings at query start for every pass of a query: [(class, geometry)]."""
    groups = pass_lanes(q_terms, df)
    cls = ring_class(len(q_terms) if len(groups) == 1 else 32, seeded)
    return [(cls, alloc_rings(cls, [int(df[t]) for t in g])) for g in groups]


# ---- corpora ----

class Lists:
    """Posting lists under construction: term → {doc: tf}."""

    def __init__(self, n_terms, n_docs):
        self.n_docs = n_docs
        self.t = [dict() for _ in range(n_terms)]

    def put(self, term, docs, tf=1):
        tfs = np.broadcast_to(np.asarray(tf), np.shape(docs))
        for d, f in zip(np.asarray(docs).tolist(), tfs.tolist()):
            self.t[term][int(d)] = int(f)

    def fill(self, rng, term, df, lo, hi, exclude=()):
        """Adds tf-1 postings at random docs in [lo, hi) until the term has df postings."""
        have = self.t[term]
        need = df - len(have)
        if need <= 0:
            return
        pool = np.setdiff1d(np.arange(lo, hi), np.fromiter(list(have) + list(exclude), np.int64))
        assert len(pool) >= need, (term, df, len(pool))
        self.put(term, np.sort(rng.choice(pool, size=need, replace=False)), 1)

    def build(self, orc):
        lists = []
        for d in self.t:
            docs = np.array(sorted(d), np.uint32)
            lists.append((docs, np.array([d[x] for x in docs.tolist()], np.uint32)))
        off = np.zeros(len(lists) + 1, np.uint64)
        off[1:] = np.cumsum([len(d) for d, _ in lists])
        post_doc = np.concatenate([d for d, _ in lists]).astype(np.uint32)
        post_tf = np.concatenate([t for _, t in lists]).astype(np.uint32)
        doc_len = np.maximum(np.bincount(post_doc, weights=post_tf, minlength=self.n_docs), 1).astype(np.uint32)
        r = restate(orc, self.n_docs, off, post_doc, post_tf, K1, B, doc_len=doc_len)
        return SimpleNamespace(n_docs=self.n_docs, n_terms=len(lists), doc_len=doc_len, post_off=off, post_doc=post_doc,
                               post_tf=post_tf, lists=lists, r=r, df=np.diff(off.astype(np.int64)))


def doc_scores(c, q):
    """Exact f64 score of every document for query q: the oracle's sum in ascending term order."""
    acc = np.zeros(c.n_docs)
    for t in sorted(int(x) for x in q):
        a, b = int(c.post_off[t]), int(c.post_off[t + 1])
        acc[c.post_doc[a:b]] = acc[c.post_doc[a:b]] + c.r.score[a:b]
    return acc


def first_window(c, lanes, al=2):
    """(hi, docs): the first chunk's window [0, hi) over the runs `lanes` and the documents any of them holds in it."""
    hi = 0xFFFFFFFF
    for t in lanes:
        d = c.lists[t][0]
        wr = min((len(d) + al - 1) & ~(al - 1), INIT)
        if wr < len(d):
            hi = min(hi, int(d[wr - 1]))
    docs = np.unique(np.concatenate([c.lists[t][0][c.lists[t][0] < hi] for t in lanes]))
    return hi, docs


def ubd(c, lanes):
    return [float(c.r.ubd[t]) for t in lanes]


def prune_at(c, lanes, Sk, ub_oth=0.0):
    """Lanes (indices into `lanes`) the prune rule takes out at threshold Sk, in the order they leave."""
    return uf.pruned_lanes(ubd(c, lanes), Sk, ub_oth)


def band(c, q, lanes, k, kp):
    """The threshold band after the first chunk: every document of the first window enters the pool (no threshold yet)
    and the pool is cut once it reaches cut_trigger entries, so the k-th score at the second chunk boundary lies between
    the lowest score in the window and its k-th highest.  Returns (S_lo, S_hi, window docs); asserts that a cut happens."""
    hi, docs = first_window(c, lanes)
    s = np.sort(doc_scores(c, q)[docs])[::-1]
    assert len(docs) >= uf.cut_trigger(k, kp, False), (len(docs), uf.cut_trigger(k, kp, False))
    return float(s[-1]), float(s[k - 1]), docs


# ---- ring-split fixture: a vocabulary of log-uniform dfs (1 .. 10^5) plus short lists, and the queries whose start
# geometry reaches every branch of alloc_rings that can be reached ----

RING_N_DOCS = 100000


def ring_vocab(seed=4101):
    rng = np.random.default_rng(seed)
    dfs = np.exp(rng.uniform(0.0, np.log(1e5), 90)).astype(np.int64)
    return np.concatenate([np.maximum(dfs, 1), rng.integers(20, 65, 40)])  # 40 short lists: the dfpad clamp of 17+ terms


def ring_queries(df, seed=4102):
    """Queries (ascending term ids) chosen greedily from random draws so that each class's start geometries, over all
    the queries of that class, take every branch that a draw reaches; the sizes the issue of fewer terms than the class
    (5 of 8, 9 of 16, 17 of 32) and one 40-term query (two groups, both split with the 32-term budget) always go in."""
    rng = np.random.default_rng(seed)
    T = len(df)
    short = np.flatnonzero(df <= 64)
    out = {"plain8": [], "plain16": [], "plain32": [], "seeded8": []}
    fixed = {"plain8": [5, 8], "plain16": [9, 16], "plain32": [17, 32, 40], "seeded8": [5, 8]}
    spans = {"plain8": (5, 8), "plain16": (9, 16), "plain32": (17, 40), "seeded8": (5, 8)}
    for cls in out:
        seen = set()
        draws = []
        for i in range(3000):
            n = int(rng.integers(spans[cls][0], spans[cls][1] + 1))
            pick = rng.choice(T, size=n, replace=False) if i % 3 else np.concatenate(
                [rng.choice(short, size=min(n - 1, len(short)), replace=False), rng.choice(T, size=1)])
            q = np.unique(pick)
            if len(q) >= spans[cls][0]:
                draws.append(q)
        for n in fixed[cls]:
            q = next(q for q in draws if len(q) == n)
            out[cls].append(q)
            seen |= branches_of(q, df, cls)
        while True:
            best = max(draws, key=lambda q: len(branches_of(q, df, cls) - seen))
            new = branches_of(best, df, cls) - seen
            if not new:
                break
            out[cls].append(best)
            seen |= new
    return out


def branches_of(q, df, cls):
    got = set()
    for _, g in query_geometries(q, df, seeded=cls == "seeded8"):
        got |= {b for b, v in g.branches.items() if v}
    return got


def ring_corpus(orc, seed=4103):
    rng = np.random.default_rng(seed)
    df = ring_vocab()
    L = Lists(len(df), RING_N_DOCS)
    for t, d in enumerate(df.tolist()):
        docs = np.sort(rng.choice(RING_N_DOCS, size=d, replace=False))
        L.put(t, docs, rng.integers(1, 6, size=d))
    return L.build(orc)


def max_halvings(cls):
    """Upper bound of the overshoot halvings of a start geometry, over every multiset of ring sizes that can overshoot.
    The rings above the floor 2^LOG_RMIN are each at most their share (rounded down; the dfpad and LOG_RMAX clamps only
    lower them), and a geometry rounded to the nearest powers of two fits by construction.  So an overshoot needs at
    least one floor ring whose share is below the floor (else Σ sizes <= Σ shares <= budget), and the list of df >= 1
    behind it leaves the other rings at most budget - 64 (a sum below the budget, of multiples of 64).  Each multiset
    that meets this is halved as the kernel does (the largest ring first) until it fits; the most halvings any of them
    needs is returned (0: the halving is unreachable)."""
    M, _, BUDGET, _, LOG_RMAX, _ = RING_CLASSES[cls]
    floor = 1 << LOG_RMIN
    sizes = [1 << l for l in range(LOG_RMIN, LOG_RMAX + 1)]

    def rec(i, left, acc):
        if i == len(sizes):
            yield acc
            return
        for c in range(left + 1):
            yield from rec(i + 1, left - c, acc + [sizes[i]] * c)

    most = 0
    for ms in rec(0, M, []):
        n_floor = ms.count(floor)  # (counting every floor ring as one below its share leaves the others the least)
        if sum(ms) <= BUDGET or n_floor == 0 or sum(ms) - n_floor * floor > BUDGET - floor:
            continue  # fits, or no floor ring below its share, or the other rings exceed what their shares allow
        ms, n = sorted(ms), 0
        while sum(ms) > BUDGET:
            ms[-1] >>= 1
            ms.sort()
            n += 1
        most = max(most, n)
    return most


# ---- prune points built on purpose ----
#
# Term roles (lanes in ascending term id):
#   S  band term: the first 32·n_S documents are "band" documents, document d held by S number d mod n_S at tf 30 — each
#      S run's 32nd posting is band document 31·n_S + i, so the first window is [0, 31·n_S) and holds band documents
#      only, all of one score B (the S terms share one df).  After the band, tf-1 postings at random.
#   H  head: tf-1 postings after the band, and one posting at tf `top` (its bound); prune candidates.
#   A  anchor: a rare term whose documents (tf 30) lift the threshold later in the query.
#   F  filler: 20 tf-1 postings on documents no other term holds (bound 8.5, above every prune sum here, and no candidate
#      it makes beats B): fills a query up to the 16- or 32-term class without changing what is pruned.
# Documents after the band: "winners" (two S terms at tf 30: score 2B, fewer than k of them; they are what a lost
# posting would drop from the rows) and "region" documents (a later, higher band that raises the threshold).

N_PRUNE = 100000


def prune_case(orc, roles, k, *, s_df=2000, n_win=6, region=None, h_avoid_s=False, seed=0):
    """roles: per lane ("S",) | ("H", df, top) | ("A", df).  region: (n_docs, holders) — n_docs documents right after the
    band holding the lanes `holders` at tf 30 (they raise the threshold above B).  h_avoid_s: the heads hold no document
    of an S term, so that no S posting and streamed head posting pass the filter together (each such candidate probes
    the pruned terms, and the probe steps count as fetched postings)."""
    rng = np.random.default_rng(seed)
    T = len(roles)
    S = [i for i, r in enumerate(roles) if r[0] == "S"]
    nS = len(S)
    W = 32 * nS
    L = Lists(T, N_PRUNE)
    for d in range(W):
        L.put(S[d % nS], [d], 30)
    reg = []
    if region:
        n_reg, holders = region
        reg = list(range(W + 50, W + 50 + 3 * n_reg, 3))
        for t in holders:
            L.put(t, reg, 30)
    win = np.linspace(W + 5000, N_PRUNE - 5000, n_win).astype(int).tolist() if n_win else []
    for j, d in enumerate(win):
        L.put(S[j % nS], [d], 30)
        L.put(S[(j + 1) % nS], [d], 30)
    fill_docs = {}
    for j, i in enumerate(i for i, r in enumerate(roles) if r[0] == "F"):
        fill_docs[i] = list(range(N_PRUNE - 1000 + 25 * j, N_PRUNE - 1000 + 25 * j + 20))
        L.put(i, fill_docs[i], 1)
    f_docs = {d for v in fill_docs.values() for d in v}
    special = set(range(W)) | set(reg) | set(win) | f_docs
    s_docs = set()
    for i in S:  # on documents of their own: no later document holds two S terms but the winners
        L.fill(rng, i, s_df, W, N_PRUNE, exclude=special | s_docs)
        s_docs |= set(L.t[i])
    for i, r in enumerate(roles):
        if r[0] == "H":
            _, df, top = r
            avoid = set(reg) | f_docs | (s_docs if h_avoid_s else set())
            if top > 1:
                L.put(i, [int(rng.choice(np.setdiff1d(np.arange(W + 100, N_PRUNE), list(avoid | special))))], top)
            L.fill(rng, i, df, W, N_PRUNE, exclude=avoid)
        elif r[0] == "A":
            L.fill(rng, i, r[1], W, N_PRUNE, exclude=special)
    c = L.build(orc)
    c.q = np.arange(T, dtype=np.uint32)
    c.k, c.roles, c.band_docs, c.region, c.winners = k, roles, W, reg, win
    return c


def prune_model(c, cls, kp):
    """What the kernel decides for a single-pass prune case: the band [S_lo, S_hi] after the first chunk, the pruned
    lanes at the second boundary (the same at both ends of the band), the final pruned set at the region's threshold,
    and in the ADAPT classes the start and re-split geometries."""
    lanes = [int(t) for t in c.q]
    S_lo, S_hi, docs = band(c, c.q, lanes, c.k, kp)
    P1 = prune_at(c, lanes, S_lo)
    out = SimpleNamespace(S_lo=S_lo, S_hi=S_hi, window=len(docs), P1=P1, P1_hi=prune_at(c, lanes, S_hi), P=P1)
    if c.region:
        s = doc_scores(c, c.q)
        top_reg = np.sort(s[c.region])[::-1]
        out.S2 = float(top_reg[c.k - 1])  # >= k region documents: the threshold after the region
        out.P = prune_at(c, lanes, out.S2)
    if cls is not None and cls in RING_CLASSES:
        dfs = [int(c.df[t]) for t in lanes]
        out.start = alloc_rings(cls, dfs)
        out.resplit = alloc_rings(cls, dfs, [i for i in range(len(lanes)) if i not in P1])
        out.moved = moved(out.start, out.resplit, [i for i in range(len(lanes)) if i not in P1])
    return out


def probe_case(orc, n_fill, n_group1=0, seed=0):
    """Block edges of a pruned (or, in a two-pass query, probed) term P.  Lanes: S1, S2 (band, df 300: B = 12.3), R (df 40:
    the candidates' term, tf 30), P (df 434 = 3 full blocks + 50, tf 1: bound 5.4 <= B / 2, pruned at the second
    boundary), then n_fill filler terms (df 50, tf 1 on documents of their own: bound 7.6, never pruned, never in the top k),
    and n_group1 more terms (df 500 .. 1000, the second group of a two-pass query together with P).  R's candidates sit
    below P's first document, on the first and last documents of its blocks, between two blocks, in the partial block,
    on P's last posting and above it; each scores 16.5 (+ 5.4 where P holds it), above every band document."""
    rng = np.random.default_rng(seed)
    S1, S2, R, P = 0, 1, 2, 3
    T = 4 + n_fill + n_group1
    L = Lists(T, N_PRUNE)
    W = 64
    for d in range(W):
        L.put(S1 if d % 2 == 0 else S2, [d], 30)
    pdocs = 1000 + 7 * np.arange(434)                 # gaps of 6 documents everywhere, also between the blocks
    L.put(P, pdocs, 1)
    blk = lambda b, i: int(pdocs[b * BLOCK + i])
    cand = dict(below=int(pdocs[0]) - 3, first0=blk(0, 0), first1=blk(1, 0), last1=blk(1, 127), last2=blk(2, 127),
                between=blk(1, 127) + 3, partial=blk(3, 20), last=int(pdocs[-1]), above=int(pdocs[-1]) + 5)
    L.put(R, sorted(cand.values()), 30)
    used = set(range(W)) | set(cand.values())
    L.fill(rng, R, 40, 20000, N_PRUNE, exclude=used)
    for t in (S1, S2):
        L.fill(rng, t, 300, 20000, N_PRUNE, exclude=used)
    for j in range(n_fill):  # disjoint documents per filler
        L.put(4 + j, 30000 + 1000 * j + np.arange(50) * 7, 1)
    for j in range(n_group1):
        L.fill(rng, 4 + n_fill + j, 500 + 60 * j, 20000, N_PRUNE, exclude=used)
    c = L.build(orc)
    c.q = np.arange(T, dtype=np.uint32)
    c.cand, c.P, c.k = cand, P, 10
    return c


def pair_case(orc, n_p=2, seed=0):
    """The block-max test and pruned terms across the two-phase launches (KEEPW classes).  Lanes: S1, S2 (df 3000; band
    B = 7.4 from single-term documents; then 40 region documents holding both at tf 30: threshold 2B), then n_p pruned
    terms (P1 and) P2 (df 45000, tf 1, bit-equal bounds c = 1.69 from one tf-30 posting each, held by Y; pruned together
    at the second boundary).  Y holds S1, S2 with 2B − n_p·c < F_S(Y) < 2B − (n_p − 1)·c: it reaches the top k only with
    every pruned term, and it is the last document of its block in P2 (the term probed first).  Z holds S1, S2 and P2 at
    tf 1 in a block of tf-1 postings only: it passes the streamed filter, and the block-max test drops it
    (F + blk_ub + rest < FloT), rightly.  n_p = 2: a 4-term query, n_p = 1: a 3-term one."""
    rng = np.random.default_rng(seed)
    S1, S2 = 0, 1
    P = list(range(2, 2 + n_p))
    P2 = P[-1]
    L = Lists(2 + n_p, N_PRUNE)
    W = 64
    for d in range(W):
        L.put(S1 if d % 2 == 0 else S2, [d], 30)
    reg = list(range(W + 50, W + 50 + 120, 3))
    for t in (S1, S2):
        L.put(t, reg, 30)
    # P2: every 2nd document from 2000 on (tf 1); Y = the last document of P2's block 40, Z inside block 60
    p2 = 2000 + 2 * np.arange(45000)
    y, z = int(p2[40 * BLOCK + 127]), int(p2[60 * BLOCK + 64])
    L.put(P2, p2, 1)
    L.put(P2, [y], 30)
    if n_p == 2:
        p1 = np.setdiff1d(1001 + 2 * np.arange(45001), [z])[:44999]
        L.put(P[0], p1, 1)
        L.put(P[0], [y], 30)
    used = set(range(W)) | set(reg) | {y, z}
    L.put(S1, [y, z], 1)
    L.put(S2, [y, z], 1)
    for t in (S1, S2):
        L.fill(rng, t, 3000, 2000, N_PRUNE, exclude=used)
    c = L.build(orc)  # the score tables (the tfs of Y and Z below change no df)
    # tfs of Y and Z on S1, S2, searched on the exact scores for the widest margins
    sc = lambda t, tf: float(c.r.s0d[t]) * tf / (tf + K1)
    B_ = sc(S1, 30)
    cb = float(c.r.ubd[P2]) / (1 + 2.0 ** -40)
    low = sc(P2, 1)
    best_y = best_z = None
    for a in range(1, 30):
        for b_ in range(1, 30):
            F = sc(S1, a) + sc(S2, b_)
            my = min(F - (2 * B_ - n_p * cb), (2 * B_ - (n_p - 1) * cb) - F)
            if best_y is None or my > best_y[0]:
                best_y = (my, a, b_)
            mz = min(F - (2 * B_ - n_p * cb), (2 * B_ - (n_p - 1) * cb - low) - F)
            if best_z is None or mz > best_z[0]:
                best_z = (mz, a, b_)
    L.put(S1, [y], best_y[1])
    L.put(S2, [y], best_y[2])
    L.put(S1, [z], best_z[1])
    L.put(S2, [z], best_z[2])
    c = L.build(orc)
    c.q = np.arange(2 + n_p, dtype=np.uint32)
    c.y, c.z, c.k, c.region, c.P = y, z, 10, reg, P
    c.margins = (best_y[0], best_z[0])
    return c


def windows(c, lanes, pruned_from, pruned, R=256, al=2, acc_docs=512, n_chunks=8, first=INIT, clamp=True):
    """The doc windows of a class of at most 8 terms (defaults: the plain kernel's fixed rings of R postings per run; the
    2..4-term classes: 8-byte rings, a 512-document dense accumulator): the first round loads `first` postings per run
    (BM25X_RING_INIT; None: a whole ring, as a seeded launch does), a window ends at the smallest last landed document of
    the runs with postings left in HBM (dense windows clamped to the accumulator when `clamp`; a seeded launch never
    clamps), and each refill tops the ring up (no top-up smaller than a quarter ring while a quarter is still unread).
    R is one size for every run or one per lane (a class that sizes its rings per query).  The lanes `pruned` (indices
    into `lanes`) leave at boundary `pruned_from` (1-based: chunk pruned_from starts without them).  Returns per chunk
    (lo, hi, rd after it), the first n_chunks chunks or (None) every chunk up to the last one (hi = INF): rd = per lane,
    postings consumed."""
    docs = [c.lists[t][0].astype(np.int64) for t in lanes]
    df = [len(d) for d in docs]
    dfpad = [(x + al - 1) & ~(al - 1) for x in df]
    R = list(R) if np.ndim(R) else [R] * len(lanes)
    wr = [min(x, R[i] if first is None else first) for i, x in enumerate(dfpad)]
    rd = [0] * len(lanes)
    lo, out = 0, []
    INF = 0xFFFFFFFF
    chunk = 0
    while n_chunks is None or chunk < n_chunks:
        chunk += 1
        act = [i for i in range(len(lanes)) if not (chunk >= pruned_from and i in pruned)]
        lim = [int(docs[i][wr[i] - 1]) for i in act if wr[i] < df[i]]
        hi = min(lim) if lim else INF
        e = {i: (min(wr[i], df[i]) if hi == INF else rd[i] + int(np.searchsorted(docs[i][rd[i]:min(wr[i], df[i])], hi)))
             for i in act}
        if clamp:
            n = [e[i] - rd[i] for i in act]
            S_, S2 = sum(n), sum(x * x for x in n)
            hi_eff = hi if hi != INF else max((int(docs[i][e[i] - 1]) + 1 for i in act if e[i] > rd[i]), default=0)
            span = max(hi_eff - lo, 0)
            if len(act) > 1 and S_ * S_ - S2 > 2 * 48 * span and span > acc_docs:
                hi = lo + acc_docs
                e = {i: rd[i] + int(np.searchsorted(docs[i][rd[i]:e[i]], hi)) for i in act}
        for i in act:
            rd[i] = e[i]
        out.append((lo, hi, list(rd)))
        lo = hi
        if hi == INF:
            break
        for i in act:
            if wr[i] < dfpad[i]:
                m = min((R[i] - (wr[i] - rd[i])) & ~(al - 1), dfpad[i] - wr[i])
                if m < R[i] // 4 and wr[i] - rd[i] >= R[i] // 4:
                    m = 0
                wr[i] += m
    return out


def two_pass_case(orc, seed=0):
    """A 40-term query whose pass 0 may prune only because of ub_oth.  Group 0 (the 32 rarest): S1, S2 (df 300, band
    B = 12.3), L1 .. L3 (df 20000, tf 1: bound 1.6 each), 27 fillers (df 100, tf 1 on documents of their own: bound 6.9,
    above B / 2).  Group 1: G1 .. G8 (df 30000; G1 .. G4 at tf 30 in X: bound 2.55 each, ub_oth = 20.4).  X holds L1 .. L3
    (tf 1) and G1 .. G4 (tf 30) and no other term: score 15 > B, in the top k.  Pass 0 without ub_oth would prune L1 .. L3
    at the second boundary; X would then hold pruned group-0 terms only, and pass 1 drops every document with a group-0 term."""
    rng = np.random.default_rng(seed)
    T = 40
    S1, S2 = 0, 1
    Ls = [2, 3, 4]
    F = list(range(5, 32))
    G = list(range(32, 40))
    L = Lists(T, N_PRUNE)
    W = 64
    for d in range(W):
        L.put(S1 if d % 2 == 0 else S2, [d], 30)
    X = [50000 + 11 * j for j in range(3)]
    for t in Ls:
        L.put(t, X, 1)
    for t in G[:4]:
        L.put(t, X, 30)
    used = set(range(W)) | set(X)
    for j, t in enumerate(F):
        L.put(t, 20000 + 100 * j + np.arange(100), 1)
        used |= set(range(20000 + 100 * j, 20100 + 100 * j))
    for t in (S1, S2):
        L.fill(rng, t, 300, 40000, N_PRUNE, exclude=used)
    for t in Ls:
        L.fill(rng, t, 20000, 2000, N_PRUNE, exclude=used)
    for t in G:
        L.fill(rng, t, 30000, 2000, N_PRUNE, exclude=used)
    c = L.build(orc)
    c.q = np.arange(T, dtype=np.uint32)
    c.X, c.k, c.Ls, c.G = X, 10, Ls, G
    return c
