"""MaxScore pruning of k_search_ring where it decides: prune sets built on purpose, the ring re-split of the 8-, 16- and
32-term classes, probes at block edges, and pruned state across passes and launches.

Every case is a corpus built from explicit lists (tests/util_prune.py, k1 = 1.2, b = 0) and a CPU model of what the
kernel decides on it; a CPU test asserts that the model reaches the decision the case is named after, and the GPU test
runs the case with pruning on and off, compares both bit for bit with OracleIndex.search_exhaustive and with each other.

  rings       alloc_rings restated for the four instantiations that split the ring budget per query (plain 8 / 16 / 32,
              seeded 8).  The fixture queries reach every branch a draw of dfs reaches (nearest / rounded-down powers of
              two, the dfpad clamp, the overshoot halving and how often, the doubling rounds), with queries shorter than
              their class and both groups of a 40-term query; an enumeration shows that the halving never runs in the
              seeded 8-term class and at most once in the plain 8-term class.  On the GPU, each class (the seeded one with nothing handed back) against the oracle.
  prune sets  the first window holds only band documents, so the threshold at the second chunk boundary lies in the
              band, and the prune set is the same at both of its ends: one head term, every term but one, bit-equal
              bounds (lowest lane first), a set that grows as the threshold rises, each shared pool size (KP 64 / 256 /
              2048).  In the ADAPT classes the re-split moves a streamed ring, and in each plain one it takes a ring past
              2^LOG_R (small_rings turns false).  The GPU asserts from bm25x_search_stats that the pruned terms' postings
              were mostly never fetched.
  probes      candidates on a pruned term's block edges (before its first document, on a block's first and last
              document, between blocks, in the partial block, on its last posting, after it) through the KEEPW probe loop
              (<= 8 terms), exact_term (16 and 32 terms) and probe_term (pass 0 of a 40-term query); the block-max test
              dropping a candidate rightly, and a candidate lifted into the top k by two pruned terms (rest / ne_prefix).
  state       a two-pass query whose pass 0 may prune only because of ub_oth; the same pruned pair across the two-phase
              launches (suspend with a non-empty pruned set, resume)."""
import numpy as np
import pytest

import util_filter as uf
import util_prune as up
from util_lib import gpu_library, set_options  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import PrefixOracle, compare, query_csr, same_rows

SEEDED8 = dict(seed=1, twophase=0, seed_max_terms=8, seed_prune_min=0xFFFFFFFF, seed_dense_div=0)
PLAIN = dict(seed=0, twophase=0)
TWOPHASE = dict(seed=0, twophase=1)

_CACHE = {}


def _cached(key, make):
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


def _oracle(orc, c):
    return orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=up.K1, b=up.B))


def _index(m, c):
    return m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=up.K1, b=up.B)


def _run_both(ix, oix, q_off, q_terms, k, opts, launches, what):
    """Pruning on and off: each against the oracle, both the same rows; returns (on, off)."""
    got = []
    for prune in (1, 0):
        set_options(ix, prune=prune, **opts)
        res = ix.search_batch(q_off, q_terms, k)
        assert res["stats"].launches == launches, (what, prune, res["stats"].launches)
        compare(res, oix, q_off, q_terms, k, what=f"{what} prune={prune}")
        got.append(res)
    same_rows(got[0], got[1], f"{what}: pruning on / off")
    return got


# ---------------------------------------------------------------------------------------------------- ring split

def _ring_fixture(orc):
    return _cached("rings", lambda: up.ring_corpus(orc))


def _ring_queries(c):
    return _cached("ring_q", lambda: up.ring_queries(c.df))


def test_ring_split_branches(orc):
    """The fixture queries reach, per class, every branch that 3000 draws of the fixture's vocabulary reach; the branch
    table (queries reaching each branch) is what the docstring of this module claims."""
    c = _ring_fixture(orc)
    qs = _ring_queries(c)
    table = {}
    for cls, queries in qs.items():
        cnt = dict.fromkeys(up.BRANCHES, 0)
        most = 0
        for q in queries:
            for _, g in up.query_geometries(q, c.df, seeded=cls == "seeded8"):
                for b, v in g.branches.items():
                    cnt[b] += int(v > 0)
                most = max(most, g.branches["halve"])
                assert g.used <= g.budget
                assert all(s == 0 or s >= 64 for s in g.size)
        table[cls] = (cnt, most)
    for cls in ("plain8", "plain16", "plain32"):
        cnt, most = table[cls]
        assert all(cnt[b] for b in ("near", "down", "clamp", "halve", "double")), (cls, cnt)
    assert table["plain16"][1] >= 2 and table["plain32"][1] >= 2, table  # halved twice in one query
    cnt, most = table["seeded8"]
    assert all(cnt[b] for b in ("near", "down", "clamp", "double")) and most == 0, cnt
    sizes = {cls: sorted({len(q) for q in qs[cls]}) for cls in qs}
    assert 5 in sizes["plain8"] and 9 in sizes["plain16"] and 17 in sizes["plain32"] and 40 in sizes["plain32"], sizes
    assert 5 in sizes["seeded8"], sizes
    # both groups of the 40-term query split the 32-term budget
    q40 = next(q for q in qs["plain32"] if len(q) == 40)
    geos = up.query_geometries(q40, c.df)
    assert len(geos) == 2 and [len([s for s in g.size if s]) for _, g in geos] == [32, 8]


def test_halving_bounds(orc):
    """How often the overshoot halving can run, by enumeration over every multiset of ring sizes (util_prune.max_halvings):
    never in the seeded 8-term class (4096 postings over at most 8 rings of 64 .. 1024), at most once in the plain 8-term
    class — both bounds the fixture queries meet — and at least as often as the fixture queries halve in the others."""
    c = _ring_fixture(orc)
    qs = _ring_queries(c)
    most = {cls: max(g.branches["halve"] for q in queries for _, g in up.query_geometries(q, c.df, seeded=cls == "seeded8"))
            for cls, queries in qs.items()}
    assert up.max_halvings("seeded8") == most["seeded8"] == 0
    assert up.max_halvings("plain8") == most["plain8"] == 1
    for cls in ("plain16", "plain32"):
        assert up.max_halvings(cls) >= most[cls] >= 2, (cls, most)


@pytest.mark.gpu
def test_ring_start_geometry(m, orc):
    """Every fixture query through its class (the 8-term one also through the seeded kernel, nothing handed back), at
    k = 10 and 100, against the oracle, pruning on and off."""
    c = _ring_fixture(orc)
    qs = _ring_queries(c)
    ix = _index(m, c)
    oix = PrefixOracle(_oracle(orc, c), 100)
    for cls, queries in qs.items():
        q_off, q_terms = query_csr(queries)
        seeded = cls == "seeded8"
        classes = {min(x for x in (8, 16, 32, 64) if x >= len(q)) for q in queries}
        for k in (10, 100):
            if seeded:  # the seeded launch's hand-back test at query start: it keeps every query
                for q in queries:
                    for prune in (1, 0):
                        assert not uf.hands_back(dict(df=c.df[q], n_docs=c.n_docs), SEEDED8, prune)
            launches = (2 if seeded else 1) * len(classes)
            _run_both(ix, oix, q_off, q_terms, k, SEEDED8 if seeded else PLAIN, launches, f"rings {cls} k={k}")
    ix.close()


# ---------------------------------------------------------------------------------------------------- prune sets

H_LOW = ("H", 80000, 1)    # bound 0.22
H_VLOW = ("H", 90000, 1)   # bound 0.105
H_HIGH = ("H", 5000, 30)   # bound 6.3: never pruned at threshold B
H_TIE = ("H", 20000, 30)   # bound 3.4: two of them do not fit under B / 2 = 4.1, one does
S = ("S",)
F = ("F",)                 # bound 8.5 on documents of its own: fills a query up to the 16- or 32-term class

# name: (roles, k, class of the ring geometry or None, KP, case keywords)
PRUNE = {
    "flip8": ([S, S] + [H_LOW] * 6, 10, "plain8", 64, {}),
    "flip16": ([S] * 4 + [H_LOW] * 12, 10, "plain16", 64, {}),
    "flip32": ([S] * 8 + [H_VLOW] * 24, 10, "plain32", 64, {}),
    "one_head4": ([S, H_LOW, S, H_HIGH], 10, None, 64, {}),
    "one_head8": ([S, H_HIGH, H_LOW, S, H_HIGH, H_HIGH], 10, "plain8", 64, {}),
    "one_head16": ([S, S, H_HIGH, H_HIGH, H_LOW, H_HIGH, H_HIGH, H_HIGH, H_HIGH], 10, "plain16", 64, {}),
    "tie8": ([S, H_TIE, S, H_TIE, H_HIGH], 10, "plain8", 64, dict(h_avoid_s=True)),
    "tie4": ([H_TIE, S, H_TIE, S], 10, None, 64, dict(h_avoid_s=True)),
    "tie16": ([S, H_TIE, S, H_TIE] + [F] * 5, 10, "plain16", 64, dict(h_avoid_s=True)),
    "tie32": ([S, H_TIE, S, H_TIE] + [F] * 13, 10, "plain32", 64, dict(h_avoid_s=True)),
    # every term but the anchor A: heads at B, then S1 and S2 (bit-equal bounds) once the A documents set the threshold
    "all_but_one8": ([S, H_VLOW, S, ("A", 40), H_VLOW, H_VLOW], 10, "plain8", 64, dict(s_df=20000, region=(40, [3]))),
    "all_but_one16": ([S, H_VLOW, S, ("A", 40)] + [H_VLOW] * 5, 10, "plain16", 64, dict(s_df=20000, region=(40, [3]))),
    # 14 heads: the 14th no longer fits under B / 2 at the second boundary, it leaves with S1 and S2
    "all_but_one32": ([S, H_VLOW, S, ("A", 40)] + [H_VLOW] * 13, 10, "plain32", 64, dict(s_df=25000, region=(40, [3]))),
    "grow8": ([S, H_LOW, S, H_HIGH], 10, "plain8", 64, dict(region=(40, [0, 2]))),
    "grow16": ([S, H_LOW, S, H_HIGH] + [F] * 5, 10, "plain16", 64, dict(region=(40, [0, 2]))),
    "grow32": ([S, H_LOW, S, H_HIGH] + [F] * 13, 10, "plain32", 64, dict(region=(40, [0, 2]))),
    "grow_kp256": ([S, S, H_LOW, S, H_HIGH], 33, "plain8", 256, dict(s_df=3000, region=(200, [0, 1]))),
    "kp2048": ([S] * 9 + [H_VLOW] * 6, 225, "plain16", 2048, dict(s_df=3000, n_win=0)),
    "resplit32_17": ([S] * 4 + [H_VLOW] * 13, 10, "plain32", 64, {}),  # fewer terms than the class
}


def _prune_fixture(orc, name):
    roles, k, cls, kp, kw = PRUNE[name]
    c = _cached(("prune", name), lambda: up.prune_case(orc, roles, k, **kw))
    return c, _cached(("prune_model", name), lambda: up.prune_model(c, cls, kp))


@pytest.mark.parametrize("name", list(PRUNE))
def test_prune_point_model(orc, name):
    """CPU: the first window holds band documents only and enough of them to cut the pool; the prune set at the second
    boundary is the same at both ends of the band; the case's own claim (below) holds."""
    roles, k, cls, kp, kw = PRUNE[name]
    c, mo = _prune_fixture(orc, name)
    assert uf.pool_capacity(k) == kp
    assert mo.P1 and mo.P1 == mo.P1_hi, (mo.P1, mo.P1_hi)
    heads = [i for i, r in enumerate(roles) if r[0] == "H" and r[2] == 1]
    if name.startswith(("flip", "kp2048", "resplit")):
        assert mo.P1 == heads or sorted(mo.P1) == heads
    if name.startswith("one_head"):
        assert len(mo.P1) == 1 and roles[mo.P1[0]] == H_LOW
    if name.startswith("tie"):
        ties = [i for i, r in enumerate(roles) if r == H_TIE]
        assert c.r.ubd[ties[0]] == c.r.ubd[ties[1]]
        assert mo.P1 == [ties[0]], mo.P1  # the lower lane of the tie, its twin stays streamed
    if "region" in kw:
        assert set(mo.P1) < set(mo.P), (mo.P1, mo.P)  # the set grows at a later boundary
        # enough region documents to cut the pool again once a threshold exists (lazy above 128 entries)
        assert len(c.region) >= uf.cut_trigger(k, kp, True) - k
    if name.startswith("grow"):
        assert [roles[i] for i in mo.P] == [H_LOW, H_HIGH], mo.P
    if name.startswith("all_but_one"):
        assert len(mo.P) == len(roles) - 1 and roles[[i for i in range(len(roles)) if i not in mo.P][0]][0] == "A"
        s_lanes = [i for i, r in enumerate(roles) if r == S]
        assert c.r.ubd[s_lanes[0]] == c.r.ubd[s_lanes[1]]
    if cls is not None:
        assert mo.moved, "the re-split moves no streamed ring"
        if name.startswith("flip"):
            assert mo.start.small and not mo.resplit.small, (mo.start.size, mo.resplit.size)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PRUNE))
def test_prune_point_gpu(m, orc, name):
    """One query, plain kernel (seed = 0 also under BM25X_SEED_FORCE=1): the oracle's rows with pruning on and off, and
    with pruning on the postings of the terms the model prunes mostly never fetched."""
    roles, k, cls, kp, kw = PRUNE[name]
    c, mo = _prune_fixture(orc, name)
    ix = _index(m, c)
    oix = _oracle(orc, c)
    q_off, q_terms = query_csr([c.q])
    on, off = _run_both(ix, oix, q_off, q_terms, k, PLAIN, 1, name)
    st_on, st_off = on["stats"], off["stats"]
    assert st_off.postings_fetched == st_off.postings
    pruned_df = sum(int(c.df[c.q[i]]) for i in mo.P)
    assert st_on.postings - st_on.postings_fetched >= pruned_df // 2, (name, st_on.postings, st_on.postings_fetched, pruned_df)
    ix.close()


# ---------------------------------------------------------------------------------------------------- probes

# name: (fillers, group-1 terms, class)
PROBE = {"keepw4": (0, 0, 4), "keepw8": (3, 0, 8), "exact16": (9, 0, 16), "exact32": (17, 0, 32), "probe_term40": (29, 7, 64)}


def _probe_fixture(orc, name):
    nf, ng, _ = PROBE[name]
    return _cached(("probe", name), lambda: up.probe_case(orc, nf, ng))


@pytest.mark.parametrize("name", list(PROBE))
def test_probe_edges_model(orc, name):
    """CPU: P has 3 full blocks and a partial one; every candidate sits where its name says; P is pruned at the second
    boundary (single pass) or probed from pass 0 (P in group 1); every candidate is in the oracle's top 40, those P holds in its top 10."""
    c = _probe_fixture(orc, name)
    P = c.P
    d = c.lists[P][0]
    assert len(d) == 3 * up.BLOCK + 50
    firsts, lasts = d[::up.BLOCK], d[up.BLOCK - 1::up.BLOCK]
    cd = c.cand
    assert cd["below"] < d[0] and cd["first0"] == d[0] and cd["first1"] == firsts[1]
    assert cd["last1"] == lasts[0 + 1] and cd["last2"] == lasts[2]
    assert lasts[1] < cd["between"] < firsts[2] and cd["between"] not in d
    assert cd["partial"] in d[3 * up.BLOCK:] and cd["last"] == d[-1] and cd["above"] > d[-1]
    groups = up.pass_lanes(c.q, c.df)
    if len(groups) == 1:
        lanes = groups[0]
        S_lo, S_hi, _ = up.band(c, c.q, lanes, c.k, 64)
        assert up.prune_at(c, lanes, S_lo) == up.prune_at(c, lanes, S_hi) == [lanes.index(P)]
    else:
        assert P in groups[1]
    od, _, _ = _oracle(orc, c).search_exhaustive(c.q, 40)
    assert set(cd.values()) <= set(od.tolist())  # in the top 40, P's holders in the top 10
    assert {v for v in cd.values() if v in d} <= set(od[:10].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PROBE))
def test_probe_edges_gpu(m, orc, name):
    c = _probe_fixture(orc, name)
    ix = _index(m, c)
    q_off, q_terms = query_csr([c.q])
    for k in (10, 40):
        _run_both(ix, _oracle(orc, c), q_off, q_terms, k, PLAIN, 1, f"{name} k={k}")
    ix.close()


PAIRS = {"pair4": 2, "pair3": 1}  # pruned terms: a 4-term query with two, a 3-term one with one


def _pair_fixture(orc, name):
    return _cached(("pair", name), lambda: up.pair_case(orc, PAIRS[name]))


def _pair_model(c):
    """Prune set at the second boundary; the chunk whose window holds the region documents (the pool is cut there, so the
    threshold is 2B at the next boundary); the suspend test of the two-phase launch at that boundary."""
    lanes = [int(t) for t in c.q]
    S_lo, S_hi, _ = up.band(c, c.q, lanes, c.k, 64)
    P1 = up.prune_at(c, lanes, S_lo)
    s = up.doc_scores(c, c.q)
    Sk2 = float(np.sort(s[c.region])[::-1][c.k - 1])
    streamed = [i for i in range(len(lanes)) if i not in P1]
    ub_ne = sum(float(c.r.ubd[lanes[i]]) for i in P1)
    Flo1, _ = uf.thresholds(S_lo, ub_ne)
    Flo, FloT = uf.thresholds(Sk2, ub_ne)
    win = up.windows(c, lanes, 2, P1)
    j = next(j for j, (_, hi, _) in enumerate(win) if max(c.region) < hi)  # chunk j + 1 consumes the last region document
    assert j >= 1  # (after the second boundary: the prune set is in place)
    lo_susp, rd = win[j + 1][0], win[j][2]
    left = sum(int(c.df[lanes[i]]) - rd[i] for i in streamed)
    return dict(S_lo=S_lo, S_hi=S_hi, P1=P1, P1_hi=up.prune_at(c, lanes, S_hi), Sk2=Sk2, Flo=Flo, FloT=FloT,
                P2=up.prune_at(c, lanes, Sk2), s=s, left=left, lo_susp=lo_susp, suspend_boundary=j + 2,
                # no suspend before: at the band's threshold a streamed term's best posting still passes alone
                solo_before=any(float(c.r.ubd[lanes[i]]) >= float(Flo1) for i in streamed),
                solo_off=all(float(c.r.ubd[lanes[i]]) < float(Flo) for i in streamed))


@pytest.mark.parametrize("name", list(PAIRS))
def test_pair_model(orc, name):
    """CPU: the pruned terms (P1 and P2: bit-equal bounds) leave at the second boundary and stay the only pruned ones at
    the region's threshold 2B.  The two-phase launch suspends at the boundary after the region's chunk, with the pruned
    set non-empty: no streamed posting can pass alone any more (it still could at the band's threshold), more than
    BM25X_SUSPEND_MIN postings are left, and Y and Z lie beyond that boundary, so the resume launch verifies them.  Y: in
    the top k, but its streamed score plus the pruned terms but one stays below FloT (only rest keeps it, block by block);
    Z: through the streamed filter (F >= Flo), dropped by the block-max test of its P2 block, and rightly so."""
    c = _pair_fixture(orc, name)
    n_p = PAIRS[name]
    mo = _pair_model(c)
    assert mo["P1"] == mo["P1_hi"] == mo["P2"] == c.P
    if n_p == 2:
        assert c.r.ubd[2] == c.r.ubd[3]
    assert mo["solo_before"] and mo["solo_off"] and mo["left"] >= up.SUSPEND_MIN, mo["left"]
    assert mo["lo_susp"] <= min(c.y, c.z), (mo["lo_susp"], mo["suspend_boundary"])
    T = len(c.q)
    P2 = c.P[-1]
    q = uf.Query(c.r.s0d[c.q], np.full(256, up.K1))
    tf = lambda d: [int(c.lists[t][1][np.searchsorted(c.lists[t][0], d)]) if d in c.lists[t][0] else 0 for t in range(T)]
    ty, tz = tf(c.y), tf(c.z)
    Fy = float(q.filter_score(ty[:2] + [0] * n_p)[1])
    Fz_lo = float(q.filter_score(tz[:2] + [0] * n_p)[0])
    Fz_hi = float(q.filter_score(tz[:2] + [0] * n_p)[1])
    rest = float(c.r.ubd[P2]) * (n_p - 1)  # the bounds of the pruned terms probed after P2
    blk = lambda d: float(c.r.blk_ub[int(c.r.blk_off[P2]) + int(np.searchsorted(c.lists[P2][0], d)) // up.BLOCK])
    i_y = int(np.searchsorted(c.lists[P2][0], c.y))
    assert i_y % up.BLOCK == up.BLOCK - 1  # Y: the last document of its P2 block
    if n_p == 2:
        assert Fy + blk(c.y) < float(mo["FloT"])  # without rest: dropped
    assert Fy + blk(c.y) + rest > float(mo["FloT"])
    assert Fz_lo >= float(mo["Flo"]) and Fz_hi + blk(c.z) + rest < float(mo["FloT"])
    assert tz[2:] == [0] * (n_p - 1) + [1]
    od, os_, _ = _oracle(orc, c).search_exhaustive(c.q, c.k)
    assert c.y in od.tolist() and c.z not in od.tolist() and mo["s"][c.z] < os_[-1]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PAIRS))
@pytest.mark.parametrize("path", ["plain", "twophase"])
def test_pair_gpu(m, orc, name, path):
    c = _pair_fixture(orc, name)
    ix = _index(m, c)
    q_off, q_terms = query_csr([c.q])
    on, _ = _run_both(ix, _oracle(orc, c), q_off, q_terms, c.k, PLAIN if path == "plain" else TWOPHASE,
                      1 if path == "plain" else 2, f"{name} {path}")
    assert c.y in on["doc"][0].tolist()
    ix.close()


# ---------------------------------------------------------------------------------------------------- two passes

def _two_pass_fixture(orc):
    return _cached("two_pass", lambda: up.two_pass_case(orc))


def test_two_pass_model(orc):
    """CPU: the first pass streams the 32 rarest terms (L1 .. L3 among them, the G terms in the second group); at the
    band's threshold the rule with ub_oth prunes nothing, without it L1 .. L3 — every group-0 term of X; X is in the top
    k and holds no other group-0 term."""
    c = _two_pass_fixture(orc)
    g0, g1 = up.pass_lanes(c.q, c.df)
    assert set(c.Ls) <= set(g0) and set(c.G) == set(g1)
    S_lo, S_hi, _ = up.band(c, c.q, g0, c.k, 64)
    ub_oth = sum(float(c.r.ubd[t]) for t in g1) * (1.0 + 1.0e-12)
    for Sk in (S_lo, S_hi):
        assert up.prune_at(c, g0, Sk, ub_oth) == []
        assert sorted(g0[i] for i in up.prune_at(c, g0, Sk)) == c.Ls
    od, _, _ = _oracle(orc, c).search_exhaustive(c.q, c.k)
    for x in c.X:
        assert x in od.tolist()
        assert [t for t in g0 if x in c.lists[t][0]] == c.Ls


@pytest.mark.gpu
def test_two_pass_gpu(m, orc):
    c = _two_pass_fixture(orc)
    ix = _index(m, c)
    q_off, q_terms = query_csr([c.q])
    on, _ = _run_both(ix, _oracle(orc, c), q_off, q_terms, c.k, PLAIN, 1, "two-pass")
    assert set(c.X) <= set(on["doc"][0].tolist())
    ix.close()
