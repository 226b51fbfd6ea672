"""GPU: `<&>` from tsvectors in one call (bm25x_evaluate_tsvectors) and evaluate on document-sharded indexes
(bm25x_evaluate_batch_sharded, bm25x_evaluate_tsvectors_sharded), bit for bit against (a) the oracle's evaluate over the
restated casts and (b) bm25x_evaluate_batch over the four-step route (tests/util_evaluate_tsvector.py):
- every keyed kind of index handle, and the refused ones (keyless, finalized replica, growing handle), out untouched;
- the merge's skip rule: unknown lexemes before, between and after known ones on both sides, duplicates, empty vectors,
  queries without positions, a merged tf >= 2^24, fieldnorm bucket edges reached through position counts;
- unknown lexemes count in the length; pair_query (one query, a permutation, NULL) and its refusals;
- sharded equals unsharded for both calls (tsvectors, keyed documents, blocks; S = 1..4; bounds; two devices; the
  sharded seal; a keyless sharded index);
- the growing segment's lexemes before and after the seal;
- eight threads on fresh handles, device memory across calls and refusals, and the sharded tables freed with the index."""
import threading

import numpy as np
import pytest

from util_cuda import D2D, cudart, free_bytes
from util_evaluate import fieldnorm_table
from util_evaluate_tsvector import (SEED, _bm, evaluate_pairs, evaluate_raw, four_step, four_step_pairs,
                                    oracle_evaluate)
from util_documents import segment
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_tsvector import assemble, cast, synthetic, write_tsvectors

pytestmark = pytest.mark.gpu


class World:
    """An index from tsvectors, the restated segment (vocabulary, oracle) and the words it was drawn from."""

    def __init__(self, m, orc, seed, n=600, k1=1.4, b=0.7, tsv=None):
        rng = np.random.default_rng(seed)
        self.words = None
        if tsv is None:
            tsv, self.words, _ = synthetic(rng, n, 5, 40, 800, 0.2)
        self.tsv, self.k1, self.b = tsv, k1, b
        self.ix = m.Index.from_tsvectors(SEED, **tsv, k1=k1, b=b)
        off, keys, tf = cast(_bm(m).intern, SEED, tsv)
        self.s = segment(off, tf, elem_key=keys)
        s = self.s
        self.oix = orc.OracleIndex(orc.Corpus(s.n_docs, s.doc_len, s.n_terms, s.post_off, s.post_doc, s.post_tf, k1, b))

    def oracle(self, m, docs, queries, pair_query=None):
        return oracle_evaluate(m, self.oix, self.s.term_keys, self.s.n_terms, docs, queries, pair_query)


def batches(rng, words, n_docs, n_queries, n_new=200):
    """Document and query tsvectors over the index's words and new ones (unknown to it), some repeated inside a vector,
    a few vectors empty; query entries with and without positions."""
    new = [bytes(rng.integers(97, 123, size=int(rng.integers(1, 30)), dtype=np.uint8)) + b"#" for _ in range(n_new)]

    def vec(n_old, n_unknown, positions):
        pick = [words[j] for j in rng.integers(0, len(words), n_old)] + [new[j] for j in rng.integers(0, n_new, n_unknown)]
        return [(x, list(range(1, int(rng.integers(1, 5)) + 1)) if positions or rng.random() < 0.5 else None) for x in pick]

    dvecs = [vec(int(rng.integers(0, 30)), int(rng.integers(0, 6)) if i % 4 else 0, True) for i in range(n_docs)]
    # query i shares up to three lexemes with document i, so that most pairs score
    qvecs = [[(x, None) for x, _ in dvecs[i % n_docs][:3]] + vec(int(rng.integers(0, 4)), int(rng.integers(0, 3)), False)
             for i in range(n_queries)]
    return write_tsvectors(dvecs), write_tsvectors(qvecs)


def check(m, w, h, docs, queries, pair_query=None, what="", sharded=False):
    """h's one call against references (a) and (b); returns the scores."""
    got = h.evaluate_tsvectors(SEED, docs, queries, pair_query)
    want = w.oracle(m, docs, queries, pair_query)
    assert np.array_equal(got, want), (what, np.flatnonzero(got != want)[:10])
    assert np.array_equal(four_step(m, h, docs, queries, pair_query, sharded), want), what
    return got


def refused_raw(m, h, docs, queries, pair_query, msg, sharded=False, code=1):
    n = len(docs["ent_off"]) - 1
    out = (0x7FF4DEADBEEF0000 + np.arange(max(n, 1), dtype=np.uint64)).view(np.float64)
    before = out.copy()
    rc, _ = evaluate_raw(m, h, docs, queries, pair_query, sharded, out=out)
    err = m.load_library().bm25x_last_error().decode()
    assert rc == code and msg in err, (rc, err, msg)
    assert np.array_equal(out.view(np.uint64), before.view(np.uint64)), f"{msg}: a refused call wrote its output"


KINDS = ["tsvectors", "documents-keyed", "blocks-doc_len", "blocks-fieldnorm"]


@pytest.mark.parametrize("kind", KINDS)
def test_handle_kinds(m, orc, kind):
    w = World(m, orc, 11)
    rng = np.random.default_rng(12)
    docs, queries = batches(rng, w.words, 400, 400)
    if kind == "tsvectors":
        h = w.ix
    elif kind == "documents-keyed":
        off, keys, tf = m.cast_tsvectors(SEED, **w.tsv)
        h = m.Index.from_documents(off, tf, elem_key=keys, k1=w.k1, b=w.b)
    else:
        args, _ = w.ix.export_blocks(doc_fieldnorm=kind == "blocks-fieldnorm", term_keys=True)
        if kind == "blocks-doc_len":
            args["doc_len"] = w.s.doc_len
        h = m.Index.from_blocks(**args)
    got = check(m, w, h, docs, queries, what=kind)
    assert np.count_nonzero(got) > 200
    if h is not w.ix:
        assert np.array_equal(w.ix.evaluate_tsvectors(SEED, docs, queries), got)
        h.close()
    w.ix.close()


def _replica(m, src):
    lay = src.layout()
    rep = m.Index.alloc_replica(lay, 0)
    rl = rep.layout()
    for i in range(len(rl.dev_ptr)):
        assert cudart().cudaMemcpy(rl.dev_ptr[i], lay.dev_ptr[i], lay.bytes[i], D2D) == 0
    rep.finalize_replica()
    return rep


def test_refused_handles(m, orc):
    """A keyless index, a finalized replica (no keys) and a bm25x_growing_create handle are refused, writing nothing."""
    w = World(m, orc, 21)
    rng = np.random.default_rng(22)
    docs, queries = batches(rng, w.words, 50, 50)
    s = w.s
    keyless = m.Index(s.n_docs, s.doc_len, s.n_terms, s.post_off, s.post_doc, s.post_tf)
    refused_raw(m, keyless.h, docs, queries, None, "bm25x_lookup_terms: index was created without term keys")
    rep = _replica(m, w.ix)
    refused_raw(m, rep.h, docs, queries, None, "bm25x_lookup_terms: index was created without term keys")
    g = w.ix.growing(np.array([0, 2], np.uint64), np.array([0, 1], np.uint32), np.array([1, 3], np.uint32),
                     doc_len=np.array([4], np.uint32))
    refused_raw(m, g.h, docs, queries, None, "bm25x_evaluate_tsvectors: the index scores with another segment's")
    # a well-formed call on the index itself still answers
    check(m, w, w.ix, docs, queries, what="sealed")
    for h in (keyless, rep, g, w.ix):
        h.close()


def _counts(items):
    """One tsvector of (lexeme, count) entries, counts up to 2^32 - 1: a count above 65 535 becomes several entries of
    the lexeme pointing at the same bytes (the cast merges them; position words are not read)."""
    area, ents = bytearray(), []
    for lex, count in items:
        full, rest = divmod(int(count), 65535)
        for c, reps in ((65535, full), (rest, 1 if rest else 0)):
            if not reps:
                continue
            at = len(area)
            area += lex + (b"\0" if len(lex) % 2 else b"") + int(c).to_bytes(2, "little")
            ents += [(at << 12) | (len(lex) << 1) | 1] * reps
    return np.frombuffer(bytes(area), np.uint8), np.array(ents, np.uint32)


def test_merge_edges(m, orc):
    """Unknown lexemes that sort before, between and after the known ones, in documents and queries: the skip rule of
    k_evaluate (a query entry >= n_terms skipped before the cursor moves, document entries >= n_terms stepped over).
    Duplicate lexemes, empty vectors, queries without positions, a merged tf >= 2^24 (scored), and documents at both
    sides of fieldnorm bucket edges reached through position counts."""
    known = [b"bb", b"dd", b"ff", b"hh", b"a-long-known-lexeme-of-thirty-b"]
    corpus = [[(x, [1, 2]) for x in known[i % 5:] + known[:i % 3]] for i in range(40)]
    w = World(m, orc, 0, tsv=write_tsvectors(corpus))
    before, between, after = b"aa", b"cc", b"zz"
    doc_rows = [
        [(before, [1]), (b"bb", [1, 2]), (between, [3]), (b"dd", [4]), (after, [5])],
        [(after, [1, 2, 3]), (b"hh", [1]), (before, [2]), (b"ff", [1, 2])],
        [(b"bb", [1]), (b"bb", [2, 3]), (between, [1]), (between, [4]), (b"dd", [5])],   # duplicates merged
        [],
        [(b"a-long-known-lexeme-of-thirty-b", [1]), (b"an-unknown-long-lexeme-of-35-bytes!", [1, 2]), (b"ff", [3])],
    ]
    q_rows = [
        [(before, None), (b"bb", None), (b"dd", None)],
        [(b"bb", None), (between, None), (b"dd", None), (after, None)],
        [(after, None), (b"ff", None), (b"hh", None), (before, [1])],
        [],
        [(b"an-unknown-long-lexeme-of-35-bytes!", None), (b"a-long-known-lexeme-of-thirty-b", None), (b"ff", None)],
    ]
    docs, queries = write_tsvectors(doc_rows), write_tsvectors(q_rows)
    n = len(doc_rows)
    all_docs = write_tsvectors([r for r in doc_rows for _ in q_rows])       # every document against every query
    got = check(m, w, w.ix, all_docs, queries, np.tile(np.arange(len(q_rows), dtype=np.uint32), n), "skip rule")
    # the first query (unknown lexeme first) against the first document matches bb and dd
    assert got[0] > 0 and got[0] == check(m, w, w.ix, docs, queries, None, "paired")[0]
    assert np.all(got[3 * len(q_rows):4 * len(q_rows)] == 0) and np.all(got[3::len(q_rows)] == 0)
    # a merged tf >= 2^24, and lengths at both sides of fieldnorm bucket edges
    table = fieldnorm_table(orc)
    vectors = [_counts([(b"bb", 300 * 65535)]), _counts([(b"dd", 1 << 24), (after, 5)])]
    for f in list(range(1, 60, 7)) + [120, 200, 255]:
        for L in (int(table[f]) - 1, int(table[f]), int(table[f]) + 1):
            if 2 <= L < (1 << 32):
                vectors.append(_counts([(b"ff", 1), (between, L - 1)]))
    big = assemble(vectors)
    one = write_tsvectors([[(b"bb", None), (b"dd", None), (b"ff", None)]])
    pq = np.zeros(len(vectors), np.uint32)
    got = check(m, w, w.ix, big, one, pq, "tf >= 2^24 and bucket edges")
    assert np.all(got > 0)
    w.ix.close()


def test_length_counts_unknown_lexemes(m, orc):
    """Dropping the unknown lexemes of a document changes its score and no other's."""
    w = World(m, orc, 31)
    rng = np.random.default_rng(32)
    known = set(w.words)
    rows, q = [], []
    for i in range(300):
        r = [(w.words[j], [1] * int(rng.integers(1, 4))) for j in rng.integers(0, len(w.words), int(rng.integers(1, 25)))]
        if i % 3:
            r += [(b"new-%d#" % int(j), [1, 2]) for j in rng.integers(0, 50, int(rng.integers(1, 4)))]
        rows.append(r)
        q.append([(x, None) for x, _ in r[:3]])
    docs, queries = write_tsvectors(rows), write_tsvectors(q)
    without = write_tsvectors([[e for e in r if e[0] in known] for r in rows])
    a = check(m, w, w.ix, docs, queries, what="with")
    b = check(m, w, w.ix, without, queries, what="without")
    has_new = np.array([i % 3 != 0 for i in range(300)])
    changed = a != b
    assert np.count_nonzero(changed & has_new) > 150 and not np.any(changed & ~has_new)


def test_pair_query(m, orc):
    w = World(m, orc, 41)
    rng = np.random.default_rng(42)
    docs, queries = batches(rng, w.words, 500, 500)
    one = write_tsvectors([[(x, None) for x in w.words[:40:3]]])
    n = 500
    every = check(m, w, w.ix, docs, one, np.zeros(n, np.uint32), "all pairs, one query")
    assert np.count_nonzero(every) > 100
    perm = rng.permutation(n).astype(np.uint32)
    by_perm = check(m, w, w.ix, docs, queries, perm, "permutation")
    plain = check(m, w, w.ix, docs, queries, None, "NULL")
    assert np.array_equal(plain, w.ix.evaluate_tsvectors(SEED, docs, queries, np.arange(n, dtype=np.uint32)))
    assert not np.array_equal(by_perm, plain)
    bad = perm.copy()
    bad[77] = n
    refused_raw(m, w.ix.h, docs, queries, bad, f"pair_query[77] = {n} is not below the {n} query tsvectors")
    refused_raw(m, w.ix.h, docs, one, None, "pair_query is NULL, but there are 1 query tsvectors for 500 document")
    w.ix.close()


def _sharded(m, w, source, S, bounds, devices):
    kw = dict(n_shards=S, doc_bounds=bounds, devices=devices)
    if source == "tsvectors":
        return m.ShardedIndex.from_tsvectors(SEED, **w.tsv, k1=w.k1, b=w.b, **kw)
    if source == "documents-keyed":
        off, keys, tf = m.cast_tsvectors(SEED, **w.tsv)
        return m.ShardedIndex.from_documents(off, tf, elem_key=keys, k1=w.k1, b=w.b, **kw)
    args, _ = w.ix.export_blocks(doc_fieldnorm=False, term_keys=True)
    args["doc_len"] = w.s.doc_len
    return m.ShardedIndex.from_blocks(**args, **kw)


def _same_both_calls(m, w, sx, docs, queries, pq, what, ix=None):
    """Both calls on the sharded index sx equal those on the unsharded index ix (w's by default) and the oracle."""
    ix = w.ix if ix is None else ix
    got = sx.evaluate_tsvectors(SEED, docs, queries, pq)
    assert np.array_equal(got, ix.evaluate_tsvectors(SEED, docs, queries, pq)), what
    assert np.array_equal(got, w.oracle(m, docs, queries, pq)), what
    pairs = four_step_pairs(m, ix, docs, queries, pq)
    rc, a = evaluate_pairs(m, sx.h, pairs, sharded=True)
    rc2, b = evaluate_pairs(m, ix.h, pairs)
    assert rc == 0 and rc2 == 0 and np.array_equal(a, b), what
    assert np.array_equal(a[:len(got)], got), what


@pytest.mark.parametrize("source", ["tsvectors", "documents-keyed", "blocks"])
def test_sharded_equals_unsharded(m, orc, source):
    w = World(m, orc, 51)
    rng = np.random.default_rng(52)
    docs, queries = batches(rng, w.words, 300, 300)
    pq = rng.integers(0, 300, 300).astype(np.uint32)
    N = w.s.n_docs
    layouts = [(S, None, None) for S in (1, 2, 3, 4)] + [(3, [0, 7, 400, N], None), (2, [0, N - 1, N], None)]
    if m.device_count() >= 2:
        layouts.append((2, None, [0, 1]))
        layouts.append((3, [0, 100, 200, N], [1, 0, 1]))
    for S, bounds, devices in layouts:
        sx = _sharded(m, w, source, S, bounds, devices)
        _same_both_calls(m, w, sx, docs, queries, pq, f"{source} S={S} bounds={bounds} devices={devices}")
        _same_both_calls(m, w, sx, docs, queries, None, f"{source} S={S} NULL")
        sx.close()
    w.ix.close()


def test_two_devices(m, orc):
    if m.device_count() < 2:
        pytest.skip("one device")
    w = World(m, orc, 55)
    rng = np.random.default_rng(56)
    docs, queries = batches(rng, w.words, 200, 200)
    sx = _sharded(m, w, "tsvectors", 2, None, [1, 0])
    _same_both_calls(m, w, sx, docs, queries, None, "shard 0 on device 1")
    sx.close()
    w.ix.close()


def test_keyless_sharded_index(m, orc):
    """The ordinal call serves a keyless sharded index; the tsvector call refuses it."""
    w = World(m, orc, 61)
    s = w.s
    kw = dict(k1=w.k1, b=w.b)
    ix = m.Index(s.n_docs, s.doc_len, s.n_terms, s.post_off, s.post_doc, s.post_tf, **kw)
    sx = m.ShardedIndex(s.n_docs, s.doc_len, s.n_terms, s.post_off, s.post_doc, s.post_tf, n_shards=3, **kw)
    rng = np.random.default_rng(62)
    docs, queries = batches(rng, w.words, 200, 200)
    pairs = four_step_pairs(m, w.ix, docs, queries, None)
    rc, a = evaluate_pairs(m, sx.h, pairs, sharded=True)
    rc2, b = evaluate_pairs(m, ix.h, pairs)
    assert rc == 0 and rc2 == 0 and np.array_equal(a, b) and np.count_nonzero(a) > 50
    refused_raw(m, sx.h, docs, queries, None, "bm25x_lookup_terms: index was created without term keys", sharded=True)
    for h in (sx, ix, w.ix):
        h.close()


def test_growing_and_seal(m, orc):
    """Lexemes inserted into a growing segment are unknown to the sealed side: they count in length and score nothing.
    After the seal (unsharded and sharded) the new index scores them, equal to the oracle over the sealed corpus."""
    w = World(m, orc, 71)
    rng = np.random.default_rng(72)
    fresh = [b"fresh-%d" % i for i in range(40)] + [b"fresh-and-long-lexeme-%d" % i for i in range(10)]
    pool = w.words[:200] + fresh
    rows = [[(pool[int(j)], [1, 2][:int(rng.integers(1, 3))]) for j in rng.integers(0, len(pool), int(rng.integers(1, 12)))]
            for _ in range(150)]
    ins = write_tsvectors(rows)
    # query i: lexemes of inserted document i, so that the seal's new terms score
    q = write_tsvectors([[(x, None) for x, _ in r[:4]] + [(pool[int(j)], None) for j in rng.integers(0, len(pool), 2)]
                         for r in rows])
    before = check(m, w, w.ix, ins, q, what="growing lexemes on the sealed side")
    sx = m.ShardedIndex.from_tsvectors(SEED, **w.tsv, k1=w.k1, b=w.b, n_shards=3)
    # the sealed corpus: the index's tsvectors then the inserted ones
    ent = np.concatenate([w.tsv["ent_off"], ins["ent_off"][1:] + w.tsv["ent_off"][-1]])
    byt = np.concatenate([w.tsv["byte_off"], ins["byte_off"][1:] + w.tsv["byte_off"][-1]])
    whole = dict(ent_off=ent, entries=np.concatenate([w.tsv["entries"], ins["entries"]]), byte_off=byt,
                 data=np.concatenate([w.tsv["data"], ins["data"]]))
    w2 = World(m, orc, 0, k1=w.k1, b=w.b, tsv=whole)
    # the seal's lengths: a sealed survivor's is the number of postings it holds (maintain.rs:356-360), a growing one's
    # its Σ tf; N, df and Σlen of the new segment follow
    s2, n0 = w2.s, w.s.n_docs
    dl = s2.doc_len.copy()
    dl[:n0] = np.bincount(w.s.post_doc, minlength=n0)
    w2.oix = orc.OracleIndex(orc.Corpus(s2.n_docs, dl, s2.n_terms, s2.post_off, s2.post_doc, s2.post_tf, w.k1, w.b))
    sealed = []
    for side in (w.ix, sx):
        seg = side.growing_segment()
        seg.insert_tsvectors(SEED, **ins)
        got = seg.seal()[0]
        seg.close()
        after = check(m, w2, got, ins, q, what=f"after the seal ({type(side).__name__})",
                      sharded=isinstance(got, m.ShardedIndex))
        assert np.count_nonzero(after != before) > 50
        sealed.append(got)
    _same_both_calls(m, w2, sealed[1], ins, q, None, "sharded seal", ix=sealed[0])
    for h in sealed + [sx, w.ix, w2.ix]:
        h.close()


def test_concurrency_and_memory(m, orc):
    """Eight threads make the first call on a fresh index and on a fresh sharded index: equal to a serial run.  After it,
    device memory is unchanged across calls and refusals; bm25x_sharded_destroy returns the sharded tables."""
    w = World(m, orc, 81)
    rng = np.random.default_rng(82)
    work = [batches(rng, w.words, 200, 200) for _ in range(8)]
    for make in (lambda: m.Index.from_tsvectors(SEED, **w.tsv, k1=w.k1, b=w.b),
                 lambda: m.ShardedIndex.from_tsvectors(SEED, **w.tsv, k1=w.k1, b=w.b, n_shards=3)):
        h = make()
        got = [None] * 8
        gate = threading.Barrier(8)

        def run(i):
            gate.wait()
            got[i] = h.evaluate_tsvectors(SEED, *work[i])

        threads = [threading.Thread(target=run, args=(i,)) for i in range(8)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for i in range(8):
            assert np.array_equal(got[i], h.evaluate_tsvectors(SEED, *work[i])), i
            assert np.array_equal(got[i], w.oracle(m, *work[i])), i
        sharded = isinstance(h, m.ShardedIndex)
        pairs = four_step_pairs(m, w.ix, *work[0], None)
        assert evaluate_pairs(m, h.h, pairs, sharded=sharded)[0] == 0
        before = free_bytes()
        docs, queries = work[1]
        no_pos = write_tsvectors([[(b"x", None)]] * (len(docs["ent_off"]) - 1))
        zero = write_tsvectors([[(b"bb", [1])]])
        zero["data"][2:4] = 0                                          # a count of 0: refused after the cast
        for _ in range(3):
            assert np.array_equal(h.evaluate_tsvectors(SEED, docs, queries), got[1])
            assert evaluate_pairs(m, h.h, pairs, sharded=sharded)[0] == 0
            refused_raw(m, h.h, no_pos, queries, None, "tsvector must have positions", sharded)
            refused_raw(m, h.h, docs, queries, np.full(len(docs["ent_off"]) - 1, 10**6, np.uint32), "pair_query[0]",
                        sharded)
            refused_raw(m, h.h, zero, write_tsvectors([[]]), None, "has position counts that sum to 0", sharded)
        assert free_bytes() == before
        h.close()
        # handles built, evaluated and closed again leave device memory where the first one left it
        after = free_bytes()
        for _ in range(2):
            h = make()
            h.evaluate_tsvectors(SEED, *work[2])
            h.close()
        assert free_bytes() == after
    w.ix.close()
