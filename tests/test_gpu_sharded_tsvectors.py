"""GPU: the document-sharded index built from tsvectors (bm25x_index_create_sharded_from_tsvectors) against the sharded
build from the restated document cast (bm25x_index_create_sharded_from_documents), shard for shard and array for array;
the shapes its passes have never run at; its query cast (bm25x_tsvector_queries_sharded) and search rows against the
unsharded tsvector index; the oracle; the golden passages; refusals across shards; the growing segment and seal over it."""
import threading

import numpy as np
import pytest

from util_cuda import free_bytes
from util_documents import segment
from util_growing_tsvector import same_arrays, same_seal
from util_index import SCALARS, check_shards
from util_lib import gpu_library, refused  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import same_rows
from util_tsvector import cast, cast_cuts, pack, pack_ids, pack_sorted, synthetic, word_table, write_tsvectors

pytestmark = pytest.mark.gpu

SEED = bytes((11 * i + 5) & 0xFF for i in range(32))
BUILD = "bm25x_index_create_sharded_from_tsvectors"
CHUNK = 1 << 22  # entries per upload chunk of the device cast (bm25x_tsvector.cu)
INFO = ("n_docs", "n_terms", "n_postings", "sum_doc_len", "avgdl", "k1", "b")


def _bm(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


def entry_bounds(ent_off, S):
    """The bounds of doc_bounds == NULL: bm25x_sharded_create's balanced rule with cum[d] = ent_off[d]."""
    cum = np.asarray(ent_off, np.int64)
    N, P = len(cum) - 1, int(cum[-1])
    b = [0]
    for s in range(1, S):
        target = (s * P + S - 1) // S
        d = b[-1] + 1 + int(np.searchsorted(cum[b[-1] + 1:], target, side="left"))
        b.append(min(d, N - (S - s)))
    return b + [N]


def concat(*batches):
    """One batch of tsvectors from several, in order."""
    ent, byt, entries, data = [np.zeros(1, np.uint64)], [np.zeros(1, np.uint64)], [], []
    for t in batches:
        ent.append(np.asarray(t["ent_off"], np.uint64)[1:] + ent[-1][-1])
        byt.append(np.asarray(t["byte_off"], np.uint64)[1:] + byt[-1][-1])
        entries.append(np.asarray(t["entries"], np.uint32))
        data.append(np.asarray(t["data"], np.uint8))
    return dict(ent_off=np.concatenate(ent), entries=np.concatenate(entries), byte_off=np.concatenate(byt),
                data=np.concatenate(data))


def _twins(m, tsv, S, keys=None, doc_bounds=None, payload=None, k1=1.2, b=0.75, devices=None):
    """The sharded tsvector build and the sharded documents build of the restated cast with the bounds it reports."""
    got = m.ShardedIndex.from_tsvectors(SEED, **tsv, payload=payload, k1=k1, b=b, n_shards=S, doc_bounds=doc_bounds,
                                        devices=devices)
    off, k, tf = cast(_bm(m).intern, SEED, tsv, keys=keys)
    want = m.ShardedIndex.from_documents(off, tf, elem_key=k, payload=payload, k1=k1, b=b, n_shards=S,
                                         doc_bounds=got.doc_bounds(), devices=devices)
    return got, want, (off, k, tf)


def _same_sharded(got, want, what):
    assert np.array_equal(got.doc_bounds(), want.doc_bounds()), f"{what}: bounds"
    a, w = got.info(), want.info()
    for f, _ in type(w)._fields_:
        assert getattr(a, f) == getattr(w, f), f"{what}: info.{f}"
    for s in range(len(want.doc_bounds()) - 1):
        lg, dg = got.shard_arrays(s)
        lw, dw = want.shard_arrays(s)
        for name in SCALARS:
            assert getattr(lg, name) == getattr(lw, name), f"{what} shard {s}: layout.{name}"
        assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min, f"{what} shard {s}"
        same_arrays(lg, dg, lw, dw, f"{what} shard {s}")


def _same_as_unsharded(m, sx, tsv, payload=None, k1=1.2, b=0.75):
    ix = m.Index.from_tsvectors(SEED, **tsv, payload=payload, k1=k1, b=b)
    a, w = sx.info(), ix.info()
    for f in INFO:
        assert getattr(a, f) == getattr(w, f), f"info.{f} differs from the unsharded index's"
    return ix


def _corpus(m, rng, n=600):
    """Synthetic tsvectors (short and long lexemes) with a run of empty ones in the middle."""
    a, _, _ = synthetic(rng, n // 2, 0, 30, 800, 0.3)
    c, _, _ = synthetic(rng, n // 2 - 20, 1, 30, 800, 0.3)
    empty = pack_ids([0] * 20, np.zeros(0, np.uint8), [0], np.zeros(0, np.int64), np.zeros(0, np.int64))
    return concat(a, empty, c)


@pytest.mark.parametrize("S", [1, 2, 3, 8, 16])
@pytest.mark.parametrize("given", [False, True])
@pytest.mark.parametrize("payload", [False, True])
def test_equals_documents_build(m, S, given, payload):
    rng = np.random.default_rng(100 * S + 10 * given + payload)
    tsv = _corpus(m, rng)
    N = len(tsv["ent_off"]) - 1
    bounds = [0] + sorted(rng.choice(np.arange(1, N), S - 1, replace=False).tolist()) + [N] if given else None
    pay = rng.integers(0, 1 << 16, 3 * N).astype(np.uint16) if payload else None
    got, want, _ = _twins(m, tsv, S, doc_bounds=bounds, payload=pay, k1=1.4, b=0.6)
    _same_sharded(got, want, f"S={S} given={given} payload={payload}")
    assert got.doc_bounds().tolist() == (bounds if given else entry_bounds(tsv["ent_off"], S))
    _same_as_unsharded(m, got, tsv, payload=pay, k1=1.4, b=0.6)


def _shapes(rng):
    """Three shards of 5 tsvectors: shard 1 all empty; a key in shard 2 only, one in every document; lexemes of 1..15
    and of 16+ bytes; duplicate lexemes the cast merges; unsorted entries."""
    long = [b"L" * 16, b"a-lexeme-longer-than-sixteen", b"q" * 200]
    vs = []
    for d in range(5):
        vs.append([(b"everywhere", [1, 2]), (b"s0-%d" % d, [1]), (long[d % 3], [3]), (b"dup", [1]), (b"dup", [4, 5])])
    vs += [[] for _ in range(5)]
    for d in range(5):
        vs.append([(b"z", [1]), (b"only-in-shard-2", [1, 2, 3][:d % 3 + 1]), (b"everywhere", [7]), (long[d % 3], [2]),
                   (long[(d + 1) % 3], [1]), (long[d % 3], [5, 6])])
    return write_tsvectors(vs)


@pytest.mark.parametrize("bounds", [[0, 5, 10, 15], None])
def test_shapes(m, bounds):
    tsv = _shapes(np.random.default_rng(1))
    got, want, (off, keys, tf) = _twins(m, tsv, 3, doc_bounds=bounds, devices=[0, 0, 0])
    _same_sharded(got, want, f"shapes bounds={bounds}")
    _same_as_unsharded(m, got, tsv)
    bm = _bm(m)
    if bounds:
        lay, _ = got.shard_arrays(1)
        assert lay.n_docs == 5 and lay.n_postings == 0, "shard 1 holds no element"
    only, every = got.lookup_terms(np.frombuffer(bm.intern(SEED, b"only-in-shard-2") + bm.intern(SEED, b"everywhere"),
                                                 np.uint8))
    ix = m.Index.from_tsvectors(SEED, **tsv)
    df = ix.df()
    assert df[only] == 5 and df[every] == 10
    # the merged duplicates: "dup" once per document with tf 1 + 2
    k_dup = np.frombuffer(bm.intern(SEED, b"dup"), np.uint8)
    at = np.flatnonzero((keys == k_dup).all(axis=1))
    assert len(at) == 5 and (tf[at] == 3).all()


def test_several_chunks_per_shard(m):
    """More than 2^22 entries in each shard (its cast and vocabulary pass run several chunks); the bound between the
    shards falls inside a chunk of the whole batch's cut loop."""
    rng = np.random.default_rng(7)
    tsv, words, wid = synthetic(rng, 90_000, 100, 130, 30_000, 0.15)
    wkeys = np.array([np.frombuffer(_bm(m).intern(SEED, w), np.uint8) for w in words])
    got, want, _ = _twins(m, tsv, 2, keys=wkeys[wid])
    _same_sharded(got, want, "chunks")
    bounds = got.doc_bounds().tolist()
    assert bounds == entry_bounds(tsv["ent_off"], 2)
    ent, byt = np.asarray(tsv["ent_off"], np.int64), np.asarray(tsv["byte_off"], np.int64)
    whole = [a for a, _, _, _ in cast_cuts(tsv)]
    assert bounds[1] not in whole, "the shard bound is a chunk start of the whole batch"
    for s in range(2):
        lo, hi = bounds[s], bounds[s + 1]
        assert ent[hi] - ent[lo] > CHUNK
        sl = dict(ent_off=ent[lo:hi + 1] - ent[lo], byte_off=byt[lo:hi + 1] - byt[lo])
        assert len([c for c in cast_cuts(sl) if c[3]]) >= 2, f"shard {s} casts in one chunk"
    _same_as_unsharded(m, got, tsv)


def _peak(build):
    """Device memory a build takes at its peak: free memory before it minus the lowest a polling thread sees."""
    before = free_bytes()
    low, done = [before], threading.Event()

    def poll():
        while not done.is_set():
            low[0] = min(low[0], free_bytes())

    t = threading.Thread(target=poll)
    t.start()
    try:
        h = build()
    finally:
        done.set()
        t.join()
    h.close()
    return before - low[0]


def test_each_shard_casts_its_own_slice(m):
    """A shard's cast holds its own entries only, not every entry up to the end of its slice: on one device, a one-tsvector
    last shard costs what a one-tsvector first shard costs (a cast sized by the slice's end would hold the batch's 20 B
    per entry twice in the first case)."""
    rng = np.random.default_rng(51)
    tsv, _, _ = synthetic(rng, 50_000, 100, 130, 30_000, 0.0)
    N, E = len(tsv["ent_off"]) - 1, len(tsv["entries"])

    def build(bounds):
        return lambda: m.ShardedIndex.from_tsvectors(SEED, **tsv, n_shards=2, doc_bounds=bounds, devices=[0, 0])

    _peak(build([0, N - 1, N]))                                     # warm-up
    last = min(_peak(build([0, N - 1, N])) for _ in range(2))
    first = min(_peak(build([0, 1, N])) for _ in range(2))
    assert abs(last - first) < 4 * E, (last, first, 20 * E)


def _query_tsvectors(rng, words, nq=300):
    pool = words[:400] + [b"unknown", b"u" * 30, b"\x00q"]
    qs = [[pool[i] for i in rng.integers(0, len(pool), int(rng.integers(0, 7)))] for _ in range(nq)]
    return pack([len(q) for q in qs], [w for q in qs for w in q], [None if rng.random() < 0.5 else 1
                                                                   for q in qs for w in q])


@pytest.mark.parametrize("S", [2, 3])
def test_queries_and_rows_equal_unsharded(m, S):
    rng = np.random.default_rng(20 + S)
    tsv, words, _ = synthetic(rng, 3000, 0, 40, 2500, 0.25)
    N = len(tsv["ent_off"]) - 1
    pay = rng.integers(0, 1 << 16, 3 * N).astype(np.uint16)
    sx = m.ShardedIndex.from_tsvectors(SEED, **tsv, payload=pay, n_shards=S)
    ix = _same_as_unsharded(m, sx, tsv, payload=pay)
    qtsv = _query_tsvectors(rng, words)
    q_off, q_terms = sx.tsvector_queries(SEED, **qtsv)
    w_off, w_terms = ix.tsvector_queries(SEED, **qtsv)
    assert np.array_equal(q_off, w_off) and np.array_equal(q_terms, w_terms)
    assert (q_terms == m.TERM_MISSING).any() and (q_terms != m.TERM_MISSING).any()
    for k in (1, 10, 100, 1000):
        same_rows(sx.search_batch(q_off, q_terms, k, want_payload=True),
                  ix.search_batch(w_off, w_terms, k, want_payload=True), f"S={S} k={k}")
    again = sx.tsvector_queries(SEED, **qtsv)   # the vocabulary already on the device
    assert np.array_equal(again[0], q_off) and np.array_equal(again[1], q_terms)


def test_shards_against_the_oracle(m, orc):
    rng = np.random.default_rng(31)
    tsv, _, _ = synthetic(rng, 400, 0, 25, 300, 0.3)
    sx = m.ShardedIndex.from_tsvectors(SEED, **tsv, n_shards=3, k1=1.4, b=0.6)
    ix = m.Index.from_tsvectors(SEED, **tsv, k1=1.4, b=0.6)
    off, keys, tf = cast(_bm(m).intern, SEED, tsv)
    check_shards(m, orc, vars(segment(off, tf, elem_key=keys)), sx, ix, 1.4, 0.6, "tsvectors S=3")


def _golden_tsvectors(golden, ids):
    docs = []
    for i in ids:
        d = {}
        for p, w in enumerate(golden["doc_lexemes"][i - 1], 1):
            d.setdefault(w.encode(), []).append(p)
        docs.append(d)
    return pack_sorted(docs)


@pytest.mark.parametrize("S", [2, 3])
def test_golden_end_to_end(m, golden, S):
    query = pack_sorted([{golden["query"].encode(): [1]}])
    for ids, rank in ((list(range(1, 11)), "ranking_full_index"), ([2, 4, 6, 8, 10], "ranking_even_ids"),
                      ([1, 3, 5, 7, 9], "ranking_odd_ids")):
        sx = m.ShardedIndex.from_tsvectors(SEED, **_golden_tsvectors(golden, ids), n_shards=S)
        assert sx.info().sum_doc_len == sum(golden["doc_lengths"][i - 1] for i in ids)
        q_off, q_terms = sx.tsvector_queries(SEED, **query)
        assert len(q_terms) == 1 and q_terms[0] != m.TERM_MISSING
        r = sx.search_batch(q_off, q_terms, 10)
        docs = r["doc"][0, :int(r["n"][0])]
        assert [ids[d] for d in docs] == golden[rank], (S, rank)
        sx.close()


def _zero_and_big():
    zero = write_tsvectors([[(b"a", [1]), (b"nopos", [])]])          # haspos with 0 positions: merged count 0
    flat, off = word_table([b"many"])
    big = pack_ids([1], flat, off, np.zeros(1, np.int64), [65535])   # 257 x 65535 positions: merged tf >= 2^24
    big["entries"] = np.repeat(big["entries"], 257)
    big["ent_off"] = np.array([0, 257], np.uint64)
    return zero, big


def _fill(n):
    return pack_sorted([{b"w%d" % i: [1]} for i in range(n)])


def test_refusal_order_across_shards(m):
    zero, big = _zero_and_big()
    two = pack_sorted([{b"x": [1]}, {b"y": [2]}])
    # 15 documents; shard 0 = 0..4 holds document 2 with a tf >= 2^24, shard 2 = 10..14 document 12 with a count of 0
    tsv = concat(two, big, _fill(9), zero, two)
    bounds = [0, 5, 10, 15]
    assert len(tsv["ent_off"]) - 1 == 15
    warm = m.ShardedIndex.from_tsvectors(SEED, **pack_sorted([{b"warm": [1]}, {b"up": [1]}]), n_shards=2)
    warm.tsvector_queries(SEED, **pack_sorted([{b"warm": [1]}]))
    m.Index.from_tsvectors(SEED, **pack_sorted([{b"warm": [1]}])).close()
    before = free_bytes()
    code, msg = refused(m, lambda: m.Index.from_tsvectors(SEED, **tsv))
    assert (code, msg) == (1, "bm25x error 1: bm25x_index_create_from_tsvectors: invalid data: a lexeme of tsvector 12 "
                              "has position counts that sum to 0")
    for S, b in ((3, bounds), (3, None), (2, [0, 11, 15])):
        got = refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **tsv, n_shards=S, doc_bounds=b))
        assert got == (code, msg.replace("bm25x_index_create_from_tsvectors", BUILD)), (S, b)
    # without the zero: the tf >= 2^24 of document 2, and of document 12 in the last shard
    for t, d in ((concat(two, big, _fill(12)), 2), (concat(two, _fill(10), big, two), 12)):
        code, msg = refused(m, lambda: m.Index.from_tsvectors(SEED, **t))
        assert code == 4 and msg.endswith(f"(document {d})")
        got = refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **t, n_shards=3, doc_bounds=bounds))
        assert got == (code, msg.replace("bm25x_index_create_from_tsvectors", BUILD)), d
    code, msg = refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **_fill(4), n_shards=2, devices=[0, 99]))
    assert code == 2 and f"{BUILD}: CUDA device 99 not available" in msg
    assert free_bytes() == before


def test_keyless_sharded_index_refused(m):
    sx = m.ShardedIndex.from_documents(np.array([0, 2, 3], np.uint64), np.array([1, 1, 2], np.uint32),
                                       elem_term=np.array([0, 1, 1], np.uint32), n_terms=2, n_shards=2)
    code, msg = refused(m, lambda: sx.tsvector_queries(SEED, **pack_sorted([{b"a": [1]}])))
    assert code == 1 and msg.endswith("bm25x_lookup_terms: index was created without term keys")


def test_growing_segment_and_seal(m):
    rng = np.random.default_rng(41)
    tsv, words, _ = synthetic(rng, 1500, 0, 30, 1200, 0.25)
    got, want, _ = _twins(m, tsv, 3)
    fresh = [b"fresh-%d" % i for i in range(50)] + [b"fresh-and-long-%d" % i for i in range(20)]
    pool = words[:300] + fresh
    ins = write_tsvectors([[(pool[int(w)], [1, 2][:int(rng.integers(1, 3))])
                            for w in rng.integers(0, len(pool), int(rng.integers(0, 12)))] for _ in range(200)])
    segs = []
    for sx in (got, want):
        seg = sx.growing_segment()
        seg.insert_tsvectors(SEED, **ins)
        seg.refresh()
        segs.append(seg)
    assert np.array_equal(segs[0].new_keys(), segs[1].new_keys())
    q = _query_tsvectors(rng, pool)
    q0, q1 = segs[0].tsvector_queries(SEED, **q), segs[1].tsvector_queries(SEED, **q)
    assert np.array_equal(q0[0], q1[0]) and np.array_equal(q0[1], q1[1])
    for k in (1, 10, 100, 1000):
        same_rows(segs[0].search_batch(*q0, k, want_payload=True), segs[1].search_batch(*q1, k, want_payload=True),
                  f"growing k={k}")
    same_seal(segs[0].seal(), segs[1].seal(), "seal")
