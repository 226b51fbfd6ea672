"""GPU: the prefilter bitmap of bm25x_search_batch where the search kernels decide.  k_search_ring tests the bitmap after
the f32 filter and before pool_insert, so every later decision (the threshold, the single-posting limit, MaxScore's prune
set, the pool cut, the two-phase hand-over) rests on what the bitmap let into the pool; and seeded_class sends a batch
with a bitmap away from the seeded kernel, whose seeds would be filtered champions that nothing replaces.  Each corpus
and bitmap is built from the CPU model of tests/util_prefilter.py, and test_prefilter_points.py asserts on the CPU that
each reaches its branch:

  champions   2-, 3-, 4- and 8-term queries whose bitmap clears the first min(k, 128) champions of one term, of every
              term, all of them but the last, or everything but the postings just past the 128-entry champion lists:
              the answer needs documents a seeded launch would never list.  Run with the seeded options forced: the
              batch must take the unseeded launches (checked by the launch count) and give the oracle's rows.
  two-phase   the 2..4-term classes with twophase = 1 (k up to 224: 129 .. 224 is served by this flavour alone), the
              hand-over placed before the decisive documents (every other one cleared: the resume launch applies the
              bitmap), after them, or never (the pool short of k, or no threshold above a single posting).
  pools       0, 1, k - 1, k and k + 1 allowed matches in every pool kind (shared KP 64 / 256 / 2048, HBM at k = 1025
              and 65 535), and k + 1 allowed matches all in the last window.
  pruning     prune_case queries of the 8-, 16- and 32-term classes: with the band allowed the head is pruned (its
              postings mostly never fetched), with it cleared nothing is (every posting fetched).
  margin      near-threshold cases whose bitmap clears the documents above A, so that the late document B decides
              against an allowed k-th (A, k = 1) a few ulps away: the plain 8-term class and the two-phase class (B
              scored by the resume launch with pruning off, by the suspend launch with pruning on).
  dense       a window the plain kernel clamps to its accumulator and sums densely, its best documents cleared.
  growing     the two-phase corpus as the sealed side of a growing segment whose decisive documents are partly cleared
              by allow_growing and partly past allow_growing_docs (whose bits are set: the cut must drop them).
  edges       an all-zero bitmap (n = 0, reset rows), an all-ones one with its padding bits set (the rows of no bitmap),
              one prepared Batch run twice (the rows of search_batch).
  shards      the champion and two-phase passes through a 3-shard ShardedIndex whose bounds cut through the decisive
              documents at offsets that are not multiples of 8.

Every case runs on every launch flavour that can take the batch (the seeded options, hand-back, dense, two-phase,
plain), pruning on and off, against OracleIndex.search_exhaustive with the same bitmap, bit for bit: doc ids, f32 and
f64 scores, counts, unused rows 0xFFFFFFFF; all flavours the same rows."""
import time

import numpy as np
import pytest

import util_prefilter as upf
import util_prune as up
from util_lib import gpu_library, set_options  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import KERNEL_PATHS, PrefixOracle, compare, query_csr, same_rows
from util_segment import growing_expect
from util_sparse import peak_host_gb

pytestmark = pytest.mark.gpu

_SEEDED = dict(KERNEL_PATHS["seeded"], seed_max_terms=8)
PATHS = dict(seeded=_SEEDED,
             handback=dict(_SEEDED, seed_prune_min=64),
             dense=dict(_SEEDED, seed_dense_div=1),
             twophase=dict(KERNEL_PATHS["twophase"], seed_max_terms=8),
             plain=dict(KERNEL_PATHS["plain"], seed_max_terms=8))
CLASSES = (1, 2, 3, 4, 8, 16, 32, 64)

_CACHE = {}


def _cached(key, make):
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.perf_counter()
    yield
    print(f"\n[prefilter points] module wall time {time.perf_counter() - t0:.1f} s, host peak {peak_host_gb():.2f} GB")


def _index(m, c, k1=up.K1):
    return m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=k1, b=up.B)


def _oracle(orc, c, kmax, k1=up.K1):
    return PrefixOracle(orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf,
                                                   k1=k1, b=up.B)), kmax)


def _launches(path, qs, k):
    """Launches of a batch with a bitmap: one per class (never the seeded launch), two for a two-phase class."""
    n = 0
    for M in sorted({min(x for x in CLASSES if x >= len(q)) for q in qs}):
        n += 2 if path == "twophase" and 2 <= M <= 4 and k <= 224 else 1
    return n


def _every_path(ix, oix, qs, k, allow, what, paths=PATHS, launches=True):
    """Every flavour, pruning on and off: the oracle's rows with the same bitmap, the same rows on every one.  Returns
    the results by (path, prune)."""
    q_off, q_terms = query_csr(qs)
    got = {}
    for name, opts in paths.items():
        for prune in (1, 0):
            set_options(ix, prune=prune, **opts)
            got[name, prune] = ix.search_batch(q_off, q_terms, k, allow=allow)
    first = next(iter(got))
    for key, res in got.items():  # the rows first: a batch on the wrong launch shows as the rows it got wrong
        compare(res, oix, q_off, q_terms, k, allow=allow, what=f"{what} {key}")
        same_rows(res, got[first], f"{what} {key} k={k}")
    if launches:
        for (name, prune), res in got.items():
            assert res["stats"].launches == _launches(name, qs, k), (what, name, prune, res["stats"].launches)
    return got


# ---------------------------------------------------------------------------------------------------- champions

def _champions(orc):
    return _cached("champions", lambda: upf.champion_case(orc))


@pytest.mark.parametrize("kind", upf.CHAMP_KINDS)
def test_filtered_champions(m, orc, kind):
    c = _champions(orc)
    ix = _index(m, c)
    oix = _oracle(orc, c, max(upf.CHAMP_KS))
    for k in upf.CHAMP_KS:
        _every_path(ix, oix, c.qs, k, upf.champion_bitmap(c, kind, k), f"champions {kind} k={k}")
    ix.close()


# ---------------------------------------------------------------------------------------------------- two-phase

def _two_phase(orc):
    return _cached("two", lambda: upf.two_phase_case(orc))


@pytest.mark.parametrize("kind", upf.TWO_KINDS)
def test_two_phase_handover(m, orc, kind):
    c = _two_phase(orc)
    ix = _index(m, c)
    oix = _oracle(orc, c, max(upf.TWO_KS))
    for k in upf.TWO_KS:
        if kind == "short" and k == 1:
            continue
        _every_path(ix, oix, c.qs, k, upf.two_phase_bitmap(c, kind, k), f"two-phase {kind} k={k}")
    ix.close()


# ---------------------------------------------------------------------------------------------------- pools

def test_unfilled_pools(m, orc):
    """Each query alone (its bitmap allows its own matches only), every pool kind; then the last-window bitmaps."""
    c = upf.pool_case(orc)
    ix = _index(m, c)
    oix = _oracle(orc, c, max(upf.POOL_KS))
    for q in c.qs:
        for k in upf.POOL_KS:
            for n in sorted({0, 1, k - 1, k, k + 1}):
                got = _every_path(ix, oix, [q], k, upf.pool_bitmap(c, q, k, n), f"pool q{len(q)} k={k} n={n}")
                assert int(got["plain", 1]["n"][0]) == min(n, k)
    q = c.qs[0]
    for k in upf.LAST_KS:
        _every_path(ix, oix, [q], k, upf.last_window_bitmap(c, q, k), f"last window k={k}")
    ix.close()


# ---------------------------------------------------------------------------------------------------- pruning

@pytest.mark.parametrize("name", list(upf.PRUNE_ROLES))
def test_prune_under_bitmap(m, orc, name):
    """The plain kernel's postings_fetched: the head's postings mostly unfetched without a bitmap and with the band
    allowed, every posting fetched with the band cleared (pruning on); every posting with pruning off."""
    c = _cached(("prune", name), lambda: upf.prune_fixture(orc, name))
    ix = _index(m, c)
    oix = _oracle(orc, c, upf.PRUNE_K)
    bms = upf.prune_bitmaps(c, upf.PRUNE_KP)
    head_df = int(c.df[c.q[c.head]])
    for label, allow in (("none", None), ("band", bms["band"]), ("cleared", bms["cleared"])):
        got = _every_path(ix, oix, [c.q], upf.PRUNE_K, allow, f"prune {name} {label}", launches=allow is not None)
        on, off = got["plain", 1]["stats"], got["plain", 0]["stats"]
        assert off.postings_fetched == off.postings, (name, label)
        if label == "cleared":
            assert on.postings_fetched == on.postings, (name, label, on.postings, on.postings_fetched)
        else:
            assert on.postings - on.postings_fetched >= head_df // 2, (name, label, on.postings, on.postings_fetched)
    ix.close()


# ---------------------------------------------------------------------------------------------------- margin

@pytest.mark.parametrize("name", list(upf.MARGIN))
def test_margin_under_bitmap(m, orc, name):
    """k = 1 with the high documents cleared: A is the allowed k-th when B is filtered; B is the answer."""
    c = _cached(("margin", name), lambda: upf.margin_case(orc, name))
    path = upf.MARGIN[name][1]
    ix = m.Index(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"], k1=2.0, b=0.0)
    oix = orc.OracleIndex(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"], c["post_tf"],
                                     k1=2.0, b=0.0))
    allow = upf.margin_bitmap(c)
    got = _every_path(ix, oix, [c["query"]], 1, allow, f"margin {name}", paths={path: PATHS[path]})
    assert got[path, 1]["doc"][0, 0] == c["b_doc"]
    ix.close()


# ---------------------------------------------------------------------------------------------------- edges

def test_bitmap_edges(m, orc):
    """All zero: n = 0 and every row reset, on every path.  All ones with the padding bits past n_docs set: exactly the
    rows without a bitmap, on every path.  One prepared Batch with a bitmap, run twice: the rows of search_batch."""
    c = _champions(orc)
    ix = _index(m, c)
    q_off, q_terms = query_csr(c.qs)
    zero = np.zeros((c.n_docs + 7) // 8, np.uint8)
    ones = upf.bitmap(c.n_docs, pad=True)
    assert c.n_docs % 8 and ones[-1] == 0xFF
    for k in (10, 129, 1025):
        for name, opts in PATHS.items():
            for prune in (1, 0):
                set_options(ix, prune=prune, **opts)
                res = ix.search_batch(q_off, q_terms, k, allow=zero)
                assert np.all(res["n"] == 0) and np.all(res["doc"] == 0xFFFFFFFF), (name, prune, k)
                same_rows(ix.search_batch(q_off, q_terms, k, allow=ones), ix.search_batch(q_off, q_terms, k),
                          f"all ones {name} prune={prune} k={k}")
    set_options(ix, prune=1, **PATHS["seeded"])
    for k in (10, 224):
        allow = upf.champion_bitmap(c, "every", k)
        want = ix.search_batch(q_off, q_terms, k, allow=allow)
        b = ix.prepare(q_off, q_terms, k, allow)
        for run in range(2):
            st = b.run()
            assert st.launches == _launches("seeded", c.qs, k)
            same_rows(b.fetch(), want, f"prepared batch run {run} k={k}")
        b.close()
    ix.close()


# ---------------------------------------------------------------------------------------------------- shards

def _sharded(m, c, decisive):
    """3 shards whose two inner bounds sit 3 and 5 documents past two decisive documents (not multiples of 8)."""
    d = sorted(decisive)
    b1, b2 = int(d[len(d) // 3]) + 3, int(d[2 * len(d) // 3]) + 5
    b1 += 1 if b1 % 8 == 0 else 0
    b2 += 1 if b2 % 8 == 0 else 0
    sx = m.ShardedIndex(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=up.K1, b=up.B, n_shards=3,
                        doc_bounds=[0, b1, b2, c.n_docs])
    return sx, (b1, b2)


def test_sharded_champions_and_two_phase(m, orc):
    """The champion bitmaps (bounds through the lead terms' replacement documents) and the two-phase ones (bounds through
    region L) at k = 10 and 128: the oracle's rows, on the plain and the seeded options."""
    paths = {p: PATHS[p] for p in ("seeded", "twophase", "plain")}
    c = _champions(orc)
    lead = np.concatenate([c.lists[q[0]][0][(c.lists[q[0]][1] <= 400 - 128) & (c.lists[q[0]][1] > 100)] for q in c.qs])
    sx, bounds = _sharded(m, c, lead)
    assert all(b % 8 for b in bounds)
    oix = _oracle(orc, c, 128)
    for kind in upf.CHAMP_KINDS:
        for k in (10, 128):
            _every_path(sx, oix, c.qs, k, upf.champion_bitmap(c, kind, k), f"sharded champions {kind} k={k}",
                        paths=paths, launches=False)
    sx.close()
    c = _two_phase(orc)
    sx, bounds = _sharded(m, c, c.L)
    assert all(b % 8 for b in bounds) and c.L[0] < bounds[0] < bounds[1] < c.L[-1]
    oix = _oracle(orc, c, 128)
    for kind in upf.TWO_KINDS:
        for k in (10, 128):
            _every_path(sx, oix, c.qs, k, upf.two_phase_bitmap(c, kind, k), f"sharded two-phase {kind} k={k}",
                        paths=paths, launches=False)
    sx.close()


# ---------------------------------------------------------------------------------------------------- dense window

def test_dense_window(m, orc):
    c = _cached("dense", lambda: upf.dense_case(orc))
    ix = _index(m, c)
    oix = _oracle(orc, c, max(upf.DENSE_KS))
    allow = upf.bitmap(c.n_docs, cleared=c.best)
    for k in upf.DENSE_KS:
        got = _every_path(ix, oix, [c.q], k, allow, f"dense window k={k}")
        assert got["plain", 1]["doc"][0, :upf.DENSE_BEST].tolist() == c.next[:k]
    ix.close()


# ---------------------------------------------------------------------------------------------------- growing

def test_growing_segment(m, orc):
    """Sealed + growing, every path of the sealed side, pruning on and off: the merged rows of the oracle's sealed scan and
    growing scan with the same bitmaps (allow_growing cut at allow_growing_docs), bit for bit."""
    c = _two_phase(orc)
    off, term, tf, doc_len, dec = upf.growing_docs(c)
    g = orc.GrowingDocs(off, term, tf, doc_len)
    oix = orc.OracleIndex(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=up.K1, b=up.B))
    ix = _index(m, c)
    seg = m.GrowingSegment(ix)
    seg.insert(off, term, tf, doc_len=doc_len)
    seg.refresh()
    ag, cut = upf.growing_bitmap(dec)
    ref = upf.growing_reference_bitmap(ag, cut)
    q_off, q_terms = query_csr(c.qs)
    for k in upf.GROW_KS:
        allow = upf.two_phase_bitmap(c, "before", k)
        want = [growing_expect(oix, g, c.n_docs, np.array(q, np.uint32), k, allow=allow, allow_g=ref) for q in c.qs]
        first = None
        for name, opts in PATHS.items():
            for prune in (1, 0):
                set_options(ix, prune=prune, **opts)
                res = seg.search_batch(q_off, q_terms, k, allow=allow, allow_growing=ag, allow_growing_docs=cut)
                what = f"growing {name} prune={prune} k={k}"
                for i, (ed, es) in enumerate(want):
                    n = int(res["n"][i])
                    assert n == len(ed) and res["doc"][i, :n].tolist() == ed, f"{what} q{i}: ids"
                    assert res["score64"][i, :n].tolist() == es, f"{what} q{i}: f64 scores"
                    assert np.array_equal(res["score"][i, :n], np.array(es).astype(np.float32)), f"{what} q{i}: f32"
                    assert np.all(res["doc"][i, n:] == 0xFFFFFFFF)
                first = first or res
                same_rows(res, first, what)
    seg.close()
    ix.close()
