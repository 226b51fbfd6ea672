"""GPU: the refresh and the seal of a growing segment on a constructed corpus, not a random one.  k_splice walks every
source of a term (refresh: the current handle's list, then the pending one; seal: the sealed list, then the growing
handle's, or the dormant list alone) in 32-posting steps with a ballot / popc compaction, each source
starting at whatever position the one before left.  TABLE chooses per term how many postings each source holds and which
of them are deleted; the documents are built from it, `coverage` derives from the built lists what every kernel step
sees (length, survivors, start position) and test_table_covers_every_case asserts the cases, so an edit that loses one
fails there.  Then every array of the refreshed handle equals bm25x_growing_create's and the CPU restatement, every array
of the seal's result equals bm25x_index_create's over util_maintain's corpus and its restatement, in both norm forms."""
from collections import namedtuple
from types import SimpleNamespace

import numpy as np
import pytest

from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_maintain import maintain
from util_segment import (MODES, World, check_result, check_searches, check_segment, docs_from_postings, first_docs,
                          pack, random_keys)

pytestmark = pytest.mark.gpu


S = (0, 1, 31, 32, 33, 64, 65)                                   # every (source, next source) pair of these lengths
L = (0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1000)          # every dormant length
EDGE = (30, 31, 32, 33, 62, 63, 64, 65)                          # ids on both sides of a bitmap word; 31 and 64 deleted
SPECIAL = 128                                                    # ids below it hold the EDGE postings only


def _span(n, lo, hi):
    i = np.arange(n)
    return (i >= lo) & (i < hi)


# which positions of a list are deleted
PATTERNS = {
    "none": lambda n: np.zeros(n, bool),
    "all": lambda n: np.ones(n, bool),
    "step": lambda n: _span(n, 32, 64),                          # the second step deleted whole
    "but_lane0": lambda n: _span(n, 33, 64),                     # ... but for its lane 0
    "but_lane31": lambda n: _span(n, 32, 63),                    # ... but for its lane 31
    "alternating": lambda n: np.arange(n) % 2 == 1,
    "ends": lambda n: _span(n, 1, n - 1),                        # only the first and the last posting kept
}

# One term: kind "live" (a sealed term with postings: its growing postings are in the segment's handle), "dead" (a sealed
# term with df 0) or "new" (an ordinal >= T) — the growing postings of the last two are dormant; sealed / old / pend =
# (length, pattern) of its sealed list, of its growing postings before the first refresh and of those after it.
# Pattern "edge": the EDGE ids and the last id of that id space.
Row = namedtuple("Row", "kind sealed old pend")


def _table():
    rows = []
    for x in S:
        for y in S:
            rows.append(Row("live", (2, "none"), (x, "none"), (y, "none")))                  # refresh: old x, pending y
            rows.append(Row("live" if x else "dead", (x, "none"), (y, "none"), (0, "none")))  # seal: sealed x, growing y
    for d in L:
        rows.append(Row("new", (0, "none"), (d - d // 2, "none"), (d // 2, "none")))
        rows.append(Row("dead", (0, "none"), (d // 3, "none"), (d - d // 3, "none")))
    for name in PATTERNS:
        for n in (96, 129):
            rows.append(Row("live", (n, name), (1, "none"), (0, "none")))                    # in the sealed list
            rows.append(Row("live", (3, "none"), (n, name), (33, "none")))                   # in the handle's list
            rows.append(Row("live", (3, "none"), (31, "none"), (n, name)))                   # in the pending list
            rows.append(Row("new", (0, "none"), (n, name), (0, "none")))                     # in the dormant list
    rows.append(Row("live", (0, "edge"), (0, "edge"), (0, "edge")))
    rows.append(Row("new", (0, "none"), (0, "edge"), (0, "edge")))
    order = {"live": 0, "dead": 0, "new": 1}
    return sorted(rows, key=lambda r: order[r.kind])             # stable: sealed terms first, in table order


TABLE = _table()

# n_sealed mod 32, n_growing mod 32, is the last sealed id / growing ordinal deleted, is the index keyed
SIZES = {"0-1": (0, 1, True, True, False), "1-31": (1, 31, False, False, True), "31-0": (31, 0, True, False, False)}
POOL = 1100                                                      # never-deleted ids the "none" lists are drawn from


class _Space:
    """One id space [lo, hi): the pattern lists take runs of their own after the special ids, the others draw from the
    never-deleted pool behind the runs; the last id belongs to the "edge" lists."""

    def __init__(self, lo, specs, mod, special):
        self.lo = lo
        self.next = lo + (SPECIAL if special else 0)
        runs = sum(n for n, p in specs if p not in ("none", "edge"))
        self.pool_lo = self.next + runs
        self.hi = self.pool_lo + POOL + 1
        while self.hi % 32 != mod:
            self.hi += 1
        self.pool = np.arange(self.pool_lo, self.hi - 1)
        self.deleted = []

    def take(self, rng, spec, edge):
        n, pattern = spec
        if pattern == "edge":
            return np.array(edge, np.int64)
        if pattern == "none":
            return np.sort(rng.choice(self.pool, size=n, replace=False))
        ids = np.arange(self.next, self.next + n)
        self.next += n
        self.deleted += ids[PATTERNS[pattern](n)].tolist()
        return ids


def build(size):
    """The corpus of TABLE at one size: per term its sealed ids and growing ordinals (those below g1 are inserted before
    the first refresh), the two deleted sets (applied after the second insert), tfs and lengths."""
    ns_mod, ng_mod, last_s, last_g, keyed = SIZES[size]
    rng = np.random.default_rng(0x57E9)
    sealed = _Space(0, [r.sealed for r in TABLE], ns_mod, True)
    old = _Space(0, [r.old for r in TABLE], 0, True)
    pend = _Space(old.hi, [r.pend for r in TABLE], ng_mod, False)
    NS, G1, NG = sealed.hi, old.hi, pend.hi
    assert (NS % 32, NG % 32) == (ns_mod, ng_mod)
    terms = []
    for r in TABLE:
        terms.append(SimpleNamespace(kind=r.kind, sealed=sealed.take(rng, r.sealed, EDGE + (NS - 1,)),
                                     old=old.take(rng, r.old, EDGE), pend=pend.take(rng, r.pend, (NG - 1,))))
    assert sealed.next == sealed.pool_lo and old.next == old.pool_lo and pend.next == pend.pool_lo
    sdel, gdel = np.zeros(NS, bool), np.zeros(NG, bool)
    sdel[sealed.deleted + [31, 64] + ([NS - 1] if last_s else [])] = True
    gdel[old.deleted + pend.deleted + [31, 64] + ([NG - 1] if last_g else [])] = True
    T = sum(r.kind != "new" for r in TABLE)
    assert all((t.kind == "new") == (i >= T) for i, t in enumerate(terms))
    assert all((t.kind == "live") == (len(t.sealed) > 0) for t in terms)
    return SimpleNamespace(NS=NS, G1=G1, NG=NG, T=T, terms=terms, sdel=sdel, gdel=gdel, keyed=keyed, rng=rng)


def _sources(c):
    """Per kernel and term, the sources in the order the kernel walks them: (name, deleted flag per posting)."""
    out = {"refresh": [], "seal": []}
    for t in c.terms:
        grow = np.r_[t.old, t.pend].astype(np.int64)
        if t.kind == "live":
            out["refresh"].append([("old", c.gdel[t.old]), ("pend", c.gdel[t.pend])])
            # the seal refreshes first: the handle's list holds the survivors only
            out["seal"].append([("sealed", c.sdel[t.sealed]), ("growing", np.zeros(int((~c.gdel[grow]).sum()), bool))])
        else:
            out["seal"].append([("dormant", c.gdel[grow])])
    return out


def coverage(c):
    """What the splice kernels meet: per source its length, survivors and start position, and per 32-posting step the
    lanes that hold a posting and those that survive."""
    seen = SimpleNamespace(pairs={"refresh": set(), "seal": set()}, dormant={"dead": set(), "new": set()}, chains=set(),
                           steps=set(), lists=set(), start=set(), one_after_boundary=set())
    src = _sources(c)
    for kernel in src:
        for chain in src[kernel]:
            if len(chain) == 2:
                seen.pairs[kernel].add((len(chain[0][1]), len(chain[1][1])))
                alive = tuple(bool((~d).sum()) for _, d in chain)
                seen.chains.add((kernel, (len(chain[0][1]) > 0,) + alive))
            pos = 0
            for name, dele in chain:
                n, keep = len(dele), ~dele
                if pos:
                    seen.start.add((name, pos % 32))
                if pos and pos % 32 == 0 and n == 1:
                    seen.one_after_boundary.add(name)
                if n and not keep.any():
                    seen.lists.add((name, "all deleted"))
                if n > 32 and keep.all():
                    seen.lists.add((name, "none deleted"))
                if n > 2 and keep[0] and keep[-1] and keep.sum() == 2:
                    seen.lists.add((name, "first and last kept"))
                for base in range(0, n, 32):
                    k = keep[base:base + 32]
                    if len(k) == 32:
                        for what, lanes in (("deleted whole", []), ("lane 0 survives", [0]), ("lane 31 survives", [31]),
                                            ("alternating", list(range(0, 32, 2)))):
                            if np.flatnonzero(k).tolist() == lanes:
                                seen.steps.add((name, what))
                pos += int(keep.sum())
    for t in c.terms:
        if t.kind != "live":
            seen.dormant[t.kind].add(len(t.old) + len(t.pend))
    return seen


@pytest.mark.parametrize("size", list(SIZES))
def test_table_covers_every_case(size):
    c = build(size)
    seen = coverage(c)
    pairs = {(x, y) for x in S for y in S}
    assert not pairs - seen.pairs["refresh"], f"(old, pending) lengths never run: {sorted(pairs - seen.pairs['refresh'])}"
    sealed_pairs = seen.pairs["seal"] | {(0, n) for n in seen.dormant["dead"]}   # sealed df 0: the postings are dormant
    assert not pairs - sealed_pairs, f"(sealed, growing) lengths never run: {sorted(pairs - sealed_pairs)}"
    for kind in ("dead", "new"):
        assert not set(L) - seen.dormant[kind], f"dormant lengths of {kind} terms: {sorted(set(L) - seen.dormant[kind])}"
    # (the first source holds postings, it has survivors, the second has survivors)
    for kernel in ("refresh", "seal"):
        for chain in ((True, True, True), (True, False, True), (True, True, False), (False, False, True)):
            if kernel == "seal" and chain == (False, False, True):
                continue    # no sealed posting: the growing ones are dormant, a chain of one source
            assert (kernel, chain) in seen.chains, f"{kernel}: no term with sources {chain}"
    assert seen.dormant["new"] - {0} and seen.dormant["dead"] - {0}
    for name in ("sealed", "dormant", "old", "pend"):
        for what in ("deleted whole", "lane 0 survives", "lane 31 survives", "alternating"):
            assert (name, what) in seen.steps, f"no step of a {name} list: {what}"
        for what in ("all deleted", "none deleted", "first and last kept"):
            assert (name, what) in seen.lists, f"no {name} list: {what}"
    assert ("growing", "none deleted") in seen.lists
    for name in ("pend", "growing"):                         # the sources that follow another one
        for pos in (0, 1, 31):
            assert (name, pos) in seen.start, f"no {name} list starts at position {pos} mod 32"
        assert name in seen.one_after_boundary, f"no {name} list of one posting after a source that ends on a step boundary"
    # deleted bits on both sides of a bitmap word, under postings, and the last id
    ns_mod, ng_mod, last_s, last_g, _ = SIZES[size]
    for name, dele, held, last in (("sealed", c.sdel, np.concatenate([t.sealed for t in c.terms]), last_s),
                                   ("growing", c.gdel, np.concatenate([np.r_[t.old, t.pend] for t in c.terms]), last_g)):
        assert set(EDGE) <= set(held.tolist()) and len(dele) - 1 in held, f"{name}: an edge id holds no posting"
        assert dele[[31, 64]].all() and not dele[[30, 32, 33, 62, 63, 65]].any(), name
        assert dele[-1] == last, name
    live = np.concatenate([np.r_[t.old, t.pend] for t in c.terms if t.kind == "live"])
    assert set(EDGE) <= set(live.tolist()) and c.NG - 1 in live     # in the handle's lists as well as the dormant ones


def _csr(lists, rng):
    """Term-major CSR of per-term ascending ids, tfs 1 .. 5."""
    off = np.zeros(len(lists) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in lists])
    doc = np.concatenate(lists).astype(np.uint32)
    return off, doc, rng.integers(1, 6, size=len(doc)).astype(np.uint32)


@pytest.mark.parametrize("form", ["doc_len", "fieldnorm"])
@pytest.mark.parametrize("size", list(SIZES))
def test_step_edges(m, orc, size, form):
    c = build(size)
    rng, with_payload = c.rng, form == "fieldnorm"
    off, doc, tf = _csr([t.sealed for t in c.terms[:c.T]], rng)
    doc_len = (np.bincount(doc, weights=tf, minlength=c.NS) + rng.integers(0, 4, size=c.NS)).astype(np.uint32)
    keys = np.array(sorted(random_keys(rng, c.T).tolist()), np.uint8) if c.keyed else None
    n_new = len(c.terms) - c.T
    new_keys = random_keys(rng, n_new, keys) if c.keyed else None
    w = World(m, c.NS, off, doc, tf, doc_len, rng.integers(0, 65536, size=(c.NS, 3)).astype(np.uint16), keys)
    g = [np.r_[t.old, t.pend] for t in c.terms]
    goff, gord, gtf = _csr(g, rng)
    docs = docs_from_postings(rng, c.NG, np.repeat(np.arange(len(g)), np.diff(goff.astype(np.int64))), gord, gtf)
    seg = w.ix.growing_segment()
    made = []
    try:
        what = f"size {size} {form}"
        seg.insert(**docs.kw(orc, form, with_payload, 0, c.G1))
        seg.refresh()
        check_segment(orc, seg, w, first_docs(docs, c.G1), form, with_payload, f"{what}, first refresh")
        seg.insert(**docs.kw(orc, form, with_payload, c.G1, c.NG))
        seg.delete(np.flatnonzero(c.gdel))
        docs.deleted[c.gdel] = 1
        seg.refresh()
        check_segment(orc, seg, w, docs, form, with_payload, f"{what}, second refresh")
        got = seg.seal(sealed_deleted=pack(c.sdel), new_keys=new_keys)
        made.append(got[0])
        r = maintain(w.n_docs, w.off, w.doc, w.tf, docs.restated(orc, form, with_payload), sealed_deleted=c.sdel,
                     sealed_payload=w.payload, sealed_keys=w.keys, new_keys=new_keys)
        check_result(m, orc, got[0], got[1:], r, f"{what}, seal")
        # a cross-check, not the bar: searches over the constructed terms
        check_searches(orc, got[0], r, rng, f"{what}, seal", ks=(1, 10, 129),
                        modes={k: MODES[k] for k in ("prune", "seed-forced")})
    finally:
        seg.close()
        for ix in made:
            ix.close()
        w.ix.close()
