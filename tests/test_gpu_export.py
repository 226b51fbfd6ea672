"""GPU: a finalized index written out as the reference's stored segment (bm25x_index_export_blocks).

Bar: every output equals, byte for byte, what flush writes for the same postings — the payloads and block directory of
the oracle's codec (oracle.EncodedBlocks), the SummaryTuple / TokenTuple pairs of the restatement in util_export (pinned
against the oracle's flush by tests/test_export.py), the norms, payloads and Σlen the index holds — for every kind of
handle; and the export feeds bm25x_index_create_from_blocks back into an index with the same arrays and rows."""
import ctypes as C
import threading
from types import SimpleNamespace

import numpy as np
import pytest

from util_corpora import BLOCK_CONFIGS
from util_cuda import D2D, cudart
from util_export import assert_export_equal, assert_summaries_match_oracle, expected_export
from util_index import fieldnorms, read_back, synthetic_payload
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_maintain import maintain
from util_parity import live_queries, same_rows
from util_segment import pack

pytestmark = pytest.mark.gpu


def _expected(orc, c, k1=1.2, b=0.75, payload=None, keys=None, fieldnorm=None, sum_len=None):
    """The export of an index over corpus c (n_docs, doc_len, post_off, post_doc, post_tf) built with these arguments."""
    if fieldnorm is None:
        fieldnorm = fieldnorms(orc, c.doc_len)
        sum_len = int(np.asarray(c.doc_len, np.uint64).sum())
    pl = np.asarray(payload, np.uint16).reshape(-1) if payload is not None else synthetic_payload(c.n_docs)
    return expected_export(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, k1, b, fieldnorm, sum_len, pl, keys)


def _keys(T):
    """Strictly ascending 16-byte keys: the ordinal big-endian, then random bytes."""
    k = np.random.default_rng(T).integers(0, 256, (T, 16), dtype=np.uint8)
    k[:, :4] = np.arange(T, dtype=">u4").view(np.uint8).reshape(T, 4)
    return k


class _Csr:
    def __init__(self, n_docs, lists, doc_len=None):
        self.n_docs, self.n_terms = int(n_docs), len(lists)
        self.post_off = np.cumsum([0] + [len(d) for d, _ in lists]).astype(np.uint64)
        self.post_doc = np.concatenate([np.asarray(d, np.uint32) for d, _ in lists])
        self.post_tf = np.concatenate([np.asarray(t, np.uint32) for _, t in lists])
        if doc_len is None:
            doc_len = np.minimum(np.bincount(self.post_doc, weights=self.post_tf, minlength=n_docs) + 1, 0xFFFFFFFF)
        self.doc_len = np.asarray(doc_len).astype(np.uint32)


def _index(m, c, **kw):
    return m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, **kw)


def _widths_corpus():
    """A little over 2^25 documents; tokens that put every codec width in play: df 1, 127, 128, 129, 255, 256, 257;
    full blocks of every doc bit width 1..26 (one delta of 2^(w-1)) and every tf bit width 1..24 (tf up to 2^24 - 1);
    short blocks of doc byte widths 1..4 (width 4 from a gap >= 2^24, standalone and as a tail) and tf byte widths 1..3;
    random tokens over the whole id range."""
    rng = np.random.default_rng(2025)
    N = (1 << 25) + 4096
    lists = []
    for df in (1, 127, 128, 129, 255, 256, 257):
        lists.append((np.sort(rng.choice(20000, df, replace=False)), rng.integers(1, 20, df)))
    for w in range(1, 27):
        deltas = np.ones(127, np.int64)
        if w > 1:
            deltas[rng.integers(0, 127)] = 1 << (w - 1)
        lists.append((int(rng.integers(0, 64)) + np.concatenate([[0], np.cumsum(deltas)]), rng.integers(1, 4, 128)))
    for w in range(1, 25):
        tf = np.ones(128, np.int64)
        tf[rng.integers(0, 128)] = (1 << w) - 1
        lists.append((np.sort(rng.choice(50000, 128, replace=False)), tf))
    for gap in (1, 200, 300, 70000, (1 << 24) + 5):
        deltas = rng.integers(1, 4, 59)
        deltas[rng.integers(0, 59)] = gap
        lists.append((int(rng.integers(0, 1000)) + np.concatenate([[0], np.cumsum(deltas)]), rng.integers(1, 9, 60)))
        head = np.sort(rng.choice(5000, 128, replace=False))
        lists.append((np.concatenate([head, 6000 + np.concatenate([[0], np.cumsum(deltas)])]), rng.integers(1, 9, 188)))
    for top in (255, 65535, (1 << 24) - 1):
        tf = rng.integers(1, top + 1, 40)
        tf[0] = top
        lists.append((np.sort(rng.choice(N, 40, replace=False)), tf))
    for _ in range(30):
        df = int(rng.integers(1, 600))
        lists.append((np.sort(rng.choice(N, df, replace=False)), rng.integers(1, 100, df)))
    return _Csr(N, lists)


@pytest.mark.parametrize("cfg", BLOCK_CONFIGS, ids=[c["name"] for c in BLOCK_CONFIGS])
def test_export_equals_the_codec(m, orc, cfg):
    c = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    ix = m.Index.from_corpus(c)
    got = ix.export_blocks()
    assert_export_equal(got, _expected(orc, c), cfg["name"])
    assert_summaries_match_oracle(orc, got, c.n_docs, c.doc_len, c.post_off, c.post_doc, c.post_tf, 1.2, 0.75, cfg["name"])
    ix.close()


@pytest.fixture(scope="module")
def widths():
    return _widths_corpus()


@pytest.mark.parametrize("keyed,with_payload", [(False, False), (True, True)])
def test_export_every_width(m, orc, widths, keyed, with_payload):
    c = widths
    payload = np.random.default_rng(7).integers(0, 1 << 16, c.n_docs * 3, dtype=np.uint16) if with_payload else None
    keys = _keys(c.n_terms) if keyed else None
    ix = _index(m, c, payload=payload, term_keys=keys)
    got = ix.export_blocks(term_keys=keyed)
    want = _expected(orc, c, payload=payload, keys=keys)
    assert_export_equal(got, want, f"keyed={keyed} payload={with_payload}")
    assert_summaries_match_oracle(orc, got, c.n_docs, c.doc_len, c.post_off, c.post_doc, c.post_tf, 1.2, 0.75, "widths")
    md, mt, n = got[0]["blk_meta_doc"], got[0]["blk_meta_tf"], got[0]["blk_n"]
    full = n == 128
    assert set(range(1, 27)) <= set(md[full].tolist()) and set(range(1, 25)) <= set(mt[full].tolist())
    assert {0x81, 0x82, 0x83, 0x84} <= set(md[~full].tolist()) and {0x81, 0x82, 0x83} <= set(mt[~full].tolist())
    assert int(got[0]["blk_wand_tf"].max()) == (1 << 24) - 1
    ix.close()


def test_export_from_every_source(m, orc):
    """bm25x_index_create (above), both stored-block ingests, a finalized replica (keys do not travel with it), a seal."""
    c = m.synth_corpus(31, 12000, 900, 4, 150, 1.0)
    want = _expected(orc, c)
    a, _ = want
    fn, total = a["doc_fieldnorm"], a["sum_doc_len"]
    common = (c.n_docs, c.n_terms, a["term_blk_off"], a["blk_min_doc"], a["blk_n"], a["blk_meta_doc"], a["blk_meta_tf"],
              a["blk_doc_off"], a["blk_tf_off"], a["data"])
    for what, ix in (("from blocks, exact lengths", m.Index.from_blocks(*common, doc_len=c.doc_len)),
                     ("from blocks, stored norms", m.Index.from_blocks(*common, doc_fieldnorm=fn, sum_doc_len=total))):
        assert_export_equal(ix.export_blocks(), want, what)
        ix.close()

    src = m.Index.from_corpus(c, term_keys=_keys(c.n_terms))
    lay = src.layout()
    rep = m.Index.alloc_replica(lay, 0)
    with pytest.raises(m.Bm25xError, match="replica not finalized"):
        rep.export_blocks()
    rl = rep.layout()
    for i in range(len(rl.dev_ptr)):
        assert cudart().cudaMemcpy(rl.dev_ptr[i], lay.dev_ptr[i], lay.bytes[i], D2D) == 0
    rep.finalize_replica()
    assert_export_equal(rep.export_blocks(), want, "finalized replica")
    with pytest.raises(m.Bm25xError, match="without term keys") as e:
        rep.export_blocks(term_keys=True)
    assert e.value.code == 1
    rep.close()

    # a seal: sealed deletes, growing inserts and deletes; its result against maintain.rs restated
    rng = np.random.default_rng(5)
    G = 700
    terms = [np.sort(rng.choice(c.n_terms + 20, int(rng.integers(0, 12)), replace=False)) for _ in range(G)]
    elem_off = np.cumsum([0] + [len(t) for t in terms]).astype(np.uint64)
    elem_term = np.concatenate(terms).astype(np.uint32)
    elem_tf = rng.integers(1, 30, len(elem_term)).astype(np.uint32)
    glen = np.array([int(elem_tf[int(elem_off[i]):int(elem_off[i + 1])].sum()) + 3 for i in range(G)], np.uint32)
    gdel = np.zeros(G, np.uint8)
    gdel[rng.choice(G, 50, replace=False)] = 1
    sdel = rng.random(c.n_docs) < 0.2
    sealed = m.Index.from_corpus(c)
    seg = sealed.growing_segment()
    seg.insert(elem_off, elem_term, elem_tf, doc_len=glen)
    seg.delete(np.flatnonzero(gdel))
    new = seg.seal(sealed_deleted=pack(sdel))[0]
    r = maintain(c.n_docs, c.post_off, c.post_doc, c.post_tf,
                 SimpleNamespace(elem_off=elem_off, elem_term=elem_term, elem_tf=elem_tf, deleted=gdel, doc_len=glen,
                                 payload=None), sealed_deleted=sdel)
    rc = _Csr(r.n_docs, [(r.post_doc[int(r.post_off[t]):int(r.post_off[t + 1])],
                          r.post_tf[int(r.post_off[t]):int(r.post_off[t + 1])]) for t in range(r.n_terms)], r.doc_len)
    got = new.export_blocks()
    assert_export_equal(got, _expected(orc, rc, payload=r.payload), "seal")
    assert_summaries_match_oracle(orc, got, rc.n_docs, rc.doc_len, rc.post_off, rc.post_doc, rc.post_tf, 1.2, 0.75, "seal")
    new.close()
    seg.close()
    sealed.close()
    src.close()


def test_round_trip(m, orc):
    """from_blocks(export(ix)) with the wand pairs: the same 13 arrays, the same derived arrays, the same rows."""
    c = m.synth_corpus(33, 40000, 3000, 8, 200, 1.0)
    payload = np.random.default_rng(3).integers(0, 1 << 16, c.n_docs * 3, dtype=np.uint16)
    ix = m.Index.from_corpus(c, payload=payload, term_keys=_keys(c.n_terms))
    args, _ = ix.export_blocks(term_keys=True)
    back = m.Index.from_blocks(**args)
    a, b = read_back(ix.layout(), ix.derived()), read_back(back.layout(), back.derived())
    for name in a:
        assert a[name].tobytes() == b[name].tobytes(), f"round trip: {name} differs"
    assert ix.info().sum_doc_len == back.info().sum_doc_len and ix.info().avgdl == back.info().avgdl
    rng = np.random.default_rng(4)
    q_off, q_terms = live_queries(rng, ix.df(), [1, 2, 3, 4, 6, 8, 12] * 20)
    for k in (10, 100):
        same_rows(ix.search_batch(q_off, q_terms, k, want_payload=True),
                  back.search_batch(q_off, q_terms, k, want_payload=True), f"round trip k={k}")
    assert np.array_equal(back.lookup_terms(_keys(c.n_terms)), np.arange(c.n_terms))
    ix.close()
    back.close()


def test_ties_take_the_earliest_posting(m, orc):
    """b = 0: tf() depends on tf alone, so every posting with the block's largest tf ties whatever its norm.  The block's
    pair must be the FIRST such posting's (norm and tf), the token's that of its first block holding the largest tf —
    with the maximum recurring in several lanes of a block (and in several positions of one lane) and across blocks."""
    rng = np.random.default_rng(11)
    N = 6000
    doc_len = rng.integers(1, 5000, N).astype(np.uint32)       # many different norms
    lists = []
    for reps in range(12):
        df = int(rng.integers(129, 700))
        d = np.sort(rng.choice(N, df, replace=False))
        tf = rng.integers(1, 6, df)
        tf[rng.choice(df, int(rng.integers(2, 9)), replace=False)] = 9     # the maximum, several times
        lists.append((d, tf))
    lists.append((np.arange(0, 512, 2), np.full(256, 4)))                 # every posting ties, across two blocks
    c = _Csr(N, lists, doc_len)
    ix = _index(m, c, b=0.0)
    got = ix.export_blocks()
    assert_export_equal(got, _expected(orc, c, b=0.0), "b = 0")
    assert_summaries_match_oracle(orc, got, c.n_docs, c.doc_len, c.post_off, c.post_doc, c.post_tf, 1.2, 0.0, "b = 0")
    fn = fieldnorms(orc, doc_len)
    a, x = got
    for t in range(c.n_terms):
        lo, hi = int(c.post_off[t]), int(c.post_off[t + 1])
        d, tf = c.post_doc[lo:hi], c.post_tf[lo:hi]
        for j, g in enumerate(range(int(a["term_blk_off"][t]), int(a["term_blk_off"][t + 1]))):
            bd, btf = d[128 * j:128 * j + 128], tf[128 * j:128 * j + 128]
            first = int(np.flatnonzero(btf == btf.max())[0])
            assert (a["blk_wand_fieldnorm"][g], a["blk_wand_tf"][g]) == (fn[bd[first]], btf.max()), (t, j)
        first = int(np.flatnonzero(tf == tf.max())[0])
        assert (x["tok_wand_fieldnorm"][t], x["tok_wand_tf"][t]) == (fn[d[first]], tf.max()), t
    ix.close()


def test_refusals(m, orc):
    c = m.synth_corpus(35, 3000, 200, 4, 60, 0.8)
    ix = m.Index.from_corpus(c)
    L = m.load_library()
    e = m.Export()
    assert L.bm25x_index_export_blocks(ix.h, C.byref(e)) == 0          # sizing call
    n_bytes = int(e.n_bytes)
    assert n_bytes == len(_expected(orc, c)[0]["data"])
    info = ix.info()
    arrays = {"blk_meta_doc": np.full(info.n_blocks, 0xAB, np.uint8), "blk_doc_off": np.full(info.n_blocks, 7, np.uint64),
              "tok_df": np.full(info.n_terms, 9, np.uint32), "doc_fieldnorm": np.full(info.n_docs, 0xCD, np.uint8),
              "bytes": np.full(n_bytes, 0xEF, np.uint8)}
    poisoned = {k: v.copy() for k, v in arrays.items()}
    e = m.Export()
    for k, v in arrays.items():
        setattr(e, k, v.ctypes.data_as(dict(m.Export._fields_)[k]))
    e.bytes_cap = n_bytes - 1
    e.sum_doc_len = 5
    assert L.bm25x_index_export_blocks(ix.h, C.byref(e)) == 1
    msg = L.bm25x_last_error().decode()
    assert str(n_bytes - 1) in msg and str(n_bytes) in msg, msg
    assert e.n_bytes == n_bytes and e.sum_doc_len == 5
    for k, v in arrays.items():
        assert np.array_equal(v, poisoned[k]), f"{k} written by a refused call"
    with pytest.raises(m.Bm25xError, match="without term keys") as err:
        ix.export_blocks(term_keys=True)
    assert err.value.code == 1
    assert L.bm25x_index_export_blocks(None, C.byref(e)) == 1
    assert L.bm25x_index_export_blocks(ix.h, None) == 1
    # a growing handle scores with the sealed segment's avgdl, not its own: its pairs would not be flush's
    g = ix.growing(np.array([0, 2, 3], np.uint64), np.array([0, 1, 1], np.uint32), np.array([1, 2, 3], np.uint32),
                   doc_len=np.array([3, 3], np.uint32))
    assert ix.info().avgdl != 3.0
    with pytest.raises(m.Bm25xError, match="another segment's statistics") as err:
        g.export_blocks()
    assert err.value.code == 1
    g.close()
    ix.close()


def test_export_while_searching(m, orc):
    """An export on its own stream while another thread searches the same handle: each gives what it gives alone."""
    c = m.synth_corpus(37, 200000, 20000, 16, 96, 1.0)
    ix = m.Index.from_corpus(c)
    q_off, q_terms = live_queries(np.random.default_rng(8), ix.df(), [1, 2, 3, 4, 8] * 400)
    rows_alone = ix.search_batch(q_off, q_terms, 10)
    exp_alone = ix.export_blocks()
    stop, seen, errors = threading.Event(), [], []

    def searcher():
        try:
            while not stop.is_set():
                seen.append(ix.search_batch(q_off, q_terms, 10))
        except Exception as ex:  # reported by the main thread
            errors.append(ex)

    th = threading.Thread(target=searcher)
    th.start()
    try:
        exports = [ix.export_blocks() for _ in range(3)]
    finally:
        stop.set()
        th.join()
    assert not errors, errors
    assert seen, "the searching thread never completed a search"
    for got in exports:
        assert_export_equal(got, exp_alone, "export beside searches")
    for r in seen:
        same_rows(r, rows_alone, "search beside an export")
    ix.close()
