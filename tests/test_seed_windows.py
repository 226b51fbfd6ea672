"""CPU: the seeded kernel's seed ↔ window hand-off (tests/util_seeds.py) and the fixtures of test_gpu_seed_windows.py.

Every fixture is asserted here to reach the branch it was built for, so that a change to a fixture or to a kernel constant
that moves a case off its branch fails without a GPU.  On every fixture the model also shows that each seed is listed in
exactly one window and that at k <= 32 no window lists more than 64 + 32·M seeds.  The generalised util_prune.windows
is pinned to what it gave its plain-kernel callers before it learnt the seeded rings."""
from types import SimpleNamespace

import numpy as np
import pytest

import util_prune as up
import util_seeds as us

_CACHE = {}


def _cached(key, make):
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


def test_plain_windows_unchanged(orc):
    """util_prune.windows with its plain-kernel defaults: the chunks test_gpu_prune_points.py reads (a pair case pruned
    at the second boundary), the same case unpruned, a probe case to its last window, and two identical lists whose
    windows are dense and clamped to the 512-document accumulator."""
    c = up.pair_case(orc, 2)
    lanes = [int(t) for t in c.q]
    bounds = [0, 62, 8436, 16354, 25191, 33741, 41761, 49695, 57943]
    rd = [[31, 31], [261, 285], [497, 539], [738, 793], [993, 1043], [1218, 1297], [1441, 1551], [1694, 1805]]
    assert up.windows(c, lanes, 2, [2, 3]) == [(bounds[i], bounds[i + 1], rd[i] + [0, 0]) for i in range(8)]
    c1 = up.pair_case(orc, 1)
    assert up.windows(c1, [int(t) for t in c1.q], 2, [2]) == [(bounds[i], bounds[i + 1], rd[i] + [0]) for i in range(8)]
    assert up.windows(c, lanes, 99, [], n_chunks=10) == [
        (0, 62, [31, 31, 0, 0]), (62, 1511, [72, 72, 255, 0]), (1511, 2019, [73, 72, 509, 10]),
        (2019, 2510, [90, 89, 755, 255]), (2510, 3018, [107, 109, 1009, 509]), (3018, 3526, [128, 127, 1263, 763]),
        (3526, 4034, [140, 143, 1517, 1017]), (4034, 4542, [159, 163, 1771, 1271]),
        (4542, 5050, [173, 182, 2025, 1525]), (5050, 5558, [188, 201, 2279, 1779])]
    p = up.probe_case(orc, 2)
    assert up.windows(p, [int(t) for t in p.q], 2, [3], n_chunks=40) == [
        (0, 62, [31, 31, 0, 0, 0, 0]), (62, 95528, [285, 284, 39, 0, 50, 50]),
        (95528, us.INF, [300, 300, 40, 0, 50, 50])]
    d = SimpleNamespace(lists=[(np.arange(0, 40000, 4),), (np.arange(0, 40000, 4),), (np.arange(1, 40000, 8),)])
    assert up.windows(d, [0, 1, 2], 99, [], n_chunks=5) == [
        (0, 124, [31, 31, 16]), (124, 636, [159, 159, 80]), (636, 1148, [287, 287, 144]), (1148, 1660, [415, 415, 208]),
        (1660, 2172, [543, 543, 272])]


def test_list_seeds_restates_the_kernel():
    """Hand-worked listings: k <= 32 lists every lane's slice in one step, whatever the count; k = 33 lists slots 0..31
    then slot 32 of each term and pauses after the slice that takes the list past 64; a lane past the live ones still
    counts its slices; a seed on hi belongs to the next window."""
    full = [list(range(40)) for _ in range(3)]
    listed, stops = us.list_seeds([s[:32] for s in full], 3, 32, 0, 100)
    assert len(listed) == 96 and stops == [] and listed[:2] == [(0, 0), (0, 1)] and listed[32] == (1, 0)
    listed, stops = us.list_seeds([s[:33] for s in full], 4, 33, 0, 100)
    assert stops == [(3, "inside")] and len(listed) == 99 and listed[32] == (0, 32) and listed[-1] == (2, 32)
    assert us.list_seeds([[5, 7]], 2, 10, 5, 7)[0] == [(0, 0)]
    _, stops = us.list_seeds([list(range(128))] * 2, 2, 128, 0, 1000)
    assert stops == [(3, "inside"), (6, "inside")]
    assert us.list_seeds([list(range(65))] * 2, 3, 65, 0, 100)[1] == [(3, "between"), (6, "between")]


@pytest.fixture(scope="module", params=[0, 1], ids=["alone", "shared"])
def full(orc, request):
    return _cached(("full", request.param), lambda: us.full_slices_case(orc, request.param))


def test_full_slices_fixture(full):
    """Each class: every term's 32 champions lie in one window of a query with four or more windows, which lists
    32·M seeds in one step at k = 32 (256 in the 8-lane class).  Alone: no other query term holds a champion document;
    shared: another one does."""
    c = full
    for q, run in zip(c.qs, c.runs):
        M = us.seeded_class(len(q))
        assert len(q) == M
        for k in c.ks:
            us.check_model(us.model(c, q, k), k)
        mo = us.model(c, q, 32)
        ws = {us.window_of(mo, j, r) for j in range(M) for r in range(32)}
        assert len(ws) == 1 and len(mo.windows) >= 4, (M, ws, len(mo.windows))
        assert len(mo.windows[ws.pop()].listed) == 32 * M
        assert all(set(us.seeds_of(c, t, 32).tolist()) <= set(run.tolist()) for t in q)
        holders = sum(np.isin(run, c.lists[t][0]).astype(int) for t in q)
        assert np.all(holders == (2 if c.shared else 1)), M


@pytest.fixture(scope="module")
def stops(orc):
    return _cached("stops", lambda: us.slice_stops_case(orc))


def test_slice_stops_fixture(stops):
    """Each (class, k): the window that holds the in-window champions lists all of them and pauses at least once for a
    verification pass; each class pauses both inside a term's slices and between two terms in one window at some k; the
    top min(k, 128) rows of each query are the last term's seeds."""
    c = stops
    both = {M: False for M in us.CLASSES}
    for q, mt in zip(c.qs, c.meta):
        mo = us.model(c, q, mt.k)
        us.check_model(mo, mt.k)
        K = min(mt.k, us.CHAMP_L)
        w = {us.window_of(mo, j, int(r)) for j in range(mt.M) for r in np.flatnonzero(mt.inm[j])}
        assert len(w) == 1, (mt.M, mt.k)
        win = mo.windows[w.pop()]
        assert len(win.listed) == sum(int(x.sum()) for x in mt.inm) and win.stops, (mt.M, mt.k)
        both[mt.M] |= {s for _, s in win.stops} == {"inside", "between"}
        s = up.doc_scores(c, q)
        top = np.lexsort((np.arange(c.n_docs), -s))[:K]
        assert set(top.tolist()) == set(us.seeds_of(c, q[-1], mt.k).tolist()), (mt.M, mt.k)
    assert all(both.values()), both


@pytest.fixture(scope="module")
def edges(orc):
    return _cached("edges", lambda: us.edge_case(orc))


def test_edge_fixture(edges):
    """Each class: term A (lane 0) lands whole in the first round and never bounds a window (the windows are the same
    without it); its slot 1 (hi - 1) and slot 2 (lo) are listed in the middle window [lo, hi), slot 0 (on hi, a document
    of the run that bounds that window) in the next one, and slots 3..9 in the last window (hi = INF), slot 3 on the
    last document."""
    c = edges
    for q, mt in zip(c.qs, c.meta):
        a = q[0]
        assert len(q) == mt.M and c.df[a] == mt.df_a <= us.ring_sizes([int(c.df[t]) for t in q])[0]
        with_a = [(lo, hi) for lo, hi, _ in us.seeded_windows(c, q)]
        R = us.ring_sizes([int(c.df[t]) for t in q])[1:]
        assert with_a == [(lo, hi) for lo, hi, _ in up.windows(c, q[1:], 1, (), R=R, al=us.AL, n_chunks=None, first=None,
                                                              clamp=False)]
        for k in us.EDGE_KS:
            us.check_model(us.model(c, q, k), k)
        mo = us.model(c, q, 10)
        assert us.seeds_of(c, a, 10).tolist() == mt.champs
        w = mo.windows[mt.w]
        assert (w.lo, w.hi) == (mt.lo, mt.hi) and 0 < mt.lo < mt.hi - 1
        assert us.window_of(mo, 0, 1) == us.window_of(mo, 0, 2) == mt.w
        assert us.window_of(mo, 0, 0) == mt.w + 1 and mo.windows[mt.w + 1].lo == mt.hi
        assert any(mt.hi in c.lists[t][0] for t in q[1:])
        assert mt.champs[3] == c.n_docs - 1
        assert all(us.window_of(mo, 0, r) == len(mo.windows) - 1 for r in range(3, 10))
        assert mo.windows[-1].hi == us.INF


@pytest.fixture(scope="module")
def reset(orc):
    return _cached("reset", lambda: us.slot_reset_case(orc))


def test_slot_reset_fixture(reset):
    """Big terms: full champion lists (df >= 128, 128 postings at tf 50); small terms: fewer postings than any limit;
    both over the same documents.  The queries alternate big and small in each class, and the model's properties hold
    on a sample of them."""
    c = reset
    assert np.all(c.df[c.big] >= us.CHAMP_L) and np.all(c.df[c.small] < min(us.RESET_KS))
    for t in c.big:
        assert np.sum(c.lists[t][1] == 50) == us.CHAMP_L
    lo = lambda ts: min(int(c.lists[t][0][0]) for t in ts)
    hi = lambda ts: max(int(c.lists[t][0][-1]) for t in ts)
    assert lo(c.big) < 100 and lo(c.small) < 2000 and hi(c.big) > c.n_docs - 100 and hi(c.small) > c.n_docs - 2000
    qs = us.reset_queries(c, 40)
    for M in us.CLASSES:
        mine = [q for q in qs if len(q) == M]
        assert len(mine) == 40 and all(set(q) <= set(c.big.tolist()) for q in mine[0::2])
        assert all(set(q) <= set(c.small.tolist()) for q in mine[1::2])
    for q in qs[::7]:
        for k in us.RESET_KS:
            us.check_model(us.model(c, q, k), k)
