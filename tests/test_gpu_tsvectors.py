"""GPU: the tsvector casts (bm25x_cast_tsvectors) against the numpy restatement of cast_tsvector_to_document /
cast_tsvector_to_query over the host bm25x_intern (tests/util_tsvector.py), bit for bit; the build from tsvectors
against the build from the restated documents; queries from tsvectors against the host lookup of the restated keys; the
golden passages end to end; device refusals that leave no memory behind."""
import numpy as np
import pytest

from util_cuda import free_bytes
from util_index import DERIVED, LAYOUT, SCALARS, read_back
from util_lib import gpu_library, refused  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import query_csr, same_rows
from util_tsvector import cast, pack, pack_ids, pack_sorted, synthetic, word_table, write_tsvectors

pytestmark = pytest.mark.gpu

SEED = bytes((7 * i + 3) & 0xFF for i in range(32))
CHUNK = 1 << 22  # entries per upload chunk of the device cast (bm25x_tsvector.cu)


def _bm(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


def _zero_byte_lexeme(m):
    """A lexeme >= 16 bytes whose keyed hash ends in a zero byte: its key comes out with the last byte patched to 1."""
    bm = _bm(m)
    for i in range(100000):
        lex = b"zero-last-byte-%d" % i
        if bm.blake3_keyed16(SEED, lex)[15] == 0:
            assert bm.intern(SEED, lex)[15] == 1
            return lex
    raise AssertionError("no lexeme found")


def _edge_vectors(m, rng):
    """Hand-made vectors: every length class of the copy and hash paths, NUL and high bytes, the zero-last-byte hash,
    repeated lexemes, empty vectors, unsorted entries."""
    def lexeme(n):
        return bytes(rng.integers(1, 256, n, dtype=np.uint8))
    vs = []
    for n in (0, 1, 15, 16, 17, 63, 64, 65, 1023, 1024, 1025, 2047):
        vs.append([(lexeme(n), [1, 2]), (b"common", [3])])
    vs.append([])
    vs.append([(b"a\x00b", [1]), (b"\x00", [2]), (b"\xff\x80\x81", [3]), (b"\x00" * 15, [4]), (b"\xff" * 15, [1]),
               (b"x" * 14 + b"\x00", [5])])
    z = _zero_byte_lexeme(m)
    vs.append([(z, [1]), (b"plain", [1, 2, 3])])
    vs.append([(b"twice", [1, 2]), (b"other", [1]), (b"twice", [5, 6, 7]), (b"w" * 40, [1]), (b"w" * 40, [9])])
    vs.append([])
    vs.append([(b"zz", [1]), (b"aa", [2]), (b"mm", [3]), (b"aa", [4])])
    vs.append([])
    return vs


def _big_vector(rng, n=100_000):
    """One vector of n entries: 1..3-byte lexemes (no NUL, some repeated), one position each."""
    lens = rng.integers(1, 4, n)
    flat = rng.integers(1, 256, int(lens.sum()), dtype=np.uint8)
    off = np.concatenate([[0], np.cumsum(lens)])
    return pack_ids([n], flat, off, np.arange(n), np.ones(n, np.int64))


def _same_cast(m, tsv, what, keys=None):
    bm = _bm(m)
    for as_query in (False, True):
        got = bm.cast_tsvectors(SEED, **tsv, as_query=as_query)
        want = cast(bm.intern, SEED, tsv, as_query=as_query, keys=keys)
        w = f"{what} query={as_query}"
        assert np.array_equal(got[0], want[0]), f"{w}: offsets"
        assert got[1].tobytes() == want[1].tobytes(), f"{w}: keys"
        assert (got[2] is None) == as_query and (as_query or np.array_equal(got[2], want[2])), f"{w}: tf"


def test_cast_edges(m):
    rng = np.random.default_rng(1)
    vs = _edge_vectors(m, rng)
    _same_cast(m, write_tsvectors(vs), "edges")
    z = _zero_byte_lexeme(m)
    off, keys, _ = _bm(m).cast_tsvectors(SEED, **write_tsvectors([[(z, [1])]]))
    assert keys[0].tobytes() == _bm(m).intern(SEED, z) and keys[0, 15] == 1


def test_cast_big_vector_and_empties(m):
    rng = np.random.default_rng(2)
    big = _big_vector(rng)
    empty = pack_ids([0, 0, 0], np.zeros(0, np.uint8), [0], np.zeros(0, np.int64), np.zeros(0, np.int64))
    _same_cast(m, big, "100k entries")
    _same_cast(m, empty, "empty vectors")


def _chunked_batch(m, seed=3):
    """More than 2^22 entries: several upload chunks, vectors straddling no chunk (chunks take whole vectors)."""
    rng = np.random.default_rng(seed)
    tsv, words, wid = synthetic(rng, 40_000, 100, 130, 30_000, 0.15)
    assert len(tsv["entries"]) > CHUNK
    wkeys = np.array([np.frombuffer(_bm(m).intern(SEED, w), np.uint8) for w in words])
    return tsv, wkeys[wid]


def test_cast_several_chunks(m):
    tsv, keys = _chunked_batch(m)
    _same_cast(m, tsv, "chunks", keys=keys)


def _same_index(got, want, what):
    lg, dg, lw, dw = got.layout(), got.derived(), want.layout(), want.derived()
    for name in SCALARS:
        assert getattr(lg, name) == getattr(lw, name), f"{what}: {name}"
    assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min, what
    ag, aw = read_back(lg, dg), read_back(lw, dw)
    for name, _ in LAYOUT + DERIVED:
        if (name in ("blk", "blk_ub") and lw.n_blocks == 0) or (name == "champ" and dw.n_champ == 0):
            continue
        assert ag[name].tobytes() == aw[name].tobytes(), f"{what}: {name} differs"
    a, w = got.info(), want.info()
    for f, _ in type(w)._fields_:
        assert getattr(a, f) == getattr(w, f), f"{what}: info.{f}"
    assert np.array_equal(got.df(), want.df()), f"{what}: df"


def _build_both(m, tsv, keys=None, payload=None, k1=1.2, b=0.75):
    off, k, tf = cast(_bm(m).intern, SEED, tsv, keys=keys)
    got = m.Index.from_tsvectors(SEED, **tsv, payload=payload, k1=k1, b=b)
    want = m.Index.from_documents(off, tf, elem_key=k, payload=payload, k1=k1, b=b)
    return got, want


def _rows(m, got, want, n_terms, what, nq=60):
    rng = np.random.default_rng(9)
    qs = [rng.choice(n_terms, size=min(n_terms, int(rng.integers(1, 9))), replace=False) for _ in range(nq)]
    q_off, q_terms = query_csr(qs)
    for k in (1, 10, 100, 1000):
        same_rows(got.search_batch(q_off, q_terms, k, want_payload=True),
                  want.search_batch(q_off, q_terms, k, want_payload=True), f"{what} k={k}")


@pytest.mark.parametrize("payload", [False, True])
def test_build_small_equals_documents(m, payload):
    rng = np.random.default_rng(4)
    vs = [v for v in _edge_vectors(m, rng)]
    tsv = write_tsvectors(vs)
    pay = rng.integers(0, 1 << 16, 3 * len(vs)).astype(np.uint16) if payload else None
    got, want = _build_both(m, tsv, payload=pay, k1=1.5, b=0.6)
    _same_index(got, want, "edges")
    _rows(m, got, want, got.n_terms, "edges")
    syn, words, wid = synthetic(rng, 3000, 0, 40, 2000, 0.3)
    pay = rng.integers(0, 1 << 16, 3 * 3000).astype(np.uint16) if payload else None
    got, want = _build_both(m, syn, payload=pay)
    _same_index(got, want, "synthetic")
    _rows(m, got, want, got.n_terms, "synthetic")


def test_build_several_chunks_equals_documents(m):
    tsv, keys = _chunked_batch(m, seed=5)
    got, want = _build_both(m, tsv, keys=keys)
    _same_index(got, want, "chunks")
    _rows(m, got, want, got.n_terms, "chunks")


def _golden_tsvectors(golden, ids):
    docs = []
    for i in ids:
        d = {}
        for p, w in enumerate(golden["doc_lexemes"][i - 1], 1):
            d.setdefault(w.encode(), []).append(p)
        docs.append(d)
    return pack_sorted(docs)


def test_golden_end_to_end(m, golden):
    query = pack_sorted([{golden["query"].encode(): [1]}])
    for ids, rank in ((list(range(1, 11)), "ranking_full_index"), ([2, 4, 6, 8, 10], "ranking_even_ids"),
                      ([1, 3, 5, 7, 9], "ranking_odd_ids")):
        ix = m.Index.from_tsvectors(SEED, **_golden_tsvectors(golden, ids))
        assert ix.info().sum_doc_len == sum(golden["doc_lengths"][i - 1] for i in ids)
        q_off, q_terms = ix.tsvector_queries(SEED, **query)
        assert len(q_terms) == 1 and q_terms[0] != m.TERM_MISSING
        r = ix.search_batch(q_off, q_terms, 10)
        docs = r["doc"][0, :int(r["n"][0])]
        assert [ids[d] for d in docs] == golden[rank], rank
        ix.close()


def test_tsvector_queries_equal_host_lookup(m):
    rng = np.random.default_rng(6)
    tsv, words, wid = synthetic(rng, 2000, 5, 30, 3000, 0.25)
    ix = m.Index.from_tsvectors(SEED, **tsv)
    bm = _bm(m)
    # queries: known words, unknown ones (short and long), repeats, empty queries
    extra = [b"unknown", b"u" * 30, b"\x00q"]
    pool = words[:500] + extra
    nq = 400
    qs = [[pool[i] for i in rng.integers(0, len(pool), int(rng.integers(0, 7)))] for _ in range(nq)]
    qtsv = pack([len(q) for q in qs], [w for q in qs for w in q], [None if rng.random() < 0.5 else 1
                                                                   for q in qs for w in q])
    q_off, q_terms = ix.tsvector_queries(SEED, **qtsv)
    off, keys, _ = cast(bm.intern, SEED, qtsv, as_query=True)
    assert np.array_equal(q_off, off.astype(np.uint32))
    want = ix.lookup_terms(keys) if len(keys) else np.zeros(0, np.uint32)
    assert np.array_equal(q_terms, want)
    assert (q_terms == m.TERM_MISSING).any() and (q_terms != m.TERM_MISSING).any()
    for k in (1, 10, 100):
        same_rows(ix.search_batch(q_off, q_terms, k), ix.search_batch(off.astype(np.uint32), want, k), f"k={k}")
    c_off = np.arange(nq + 1, dtype=np.uint32) * 50
    c_docs = rng.integers(0, 2000, nq * 50).astype(np.uint32)
    same_rows(ix.search_candidates(q_off, q_terms, c_off, c_docs, 10),
              ix.search_candidates(off.astype(np.uint32), want, c_off, c_docs, 10), "candidates")
    # a handle whose vocabulary is already on the device: the same again
    q2 = ix.tsvector_queries(SEED, **qtsv)
    assert np.array_equal(q2[0], q_off) and np.array_equal(q2[1], q_terms)


def test_keyless_index_refused(m):
    ix = m.Index.from_documents(np.array([0, 2], np.uint64), np.array([1, 1], np.uint32),
                                elem_term=np.array([0, 1], np.uint32), n_terms=2)
    code, msg = refused(m, lambda: ix.tsvector_queries(SEED, **pack_sorted([{b"a": [1]}])))
    assert code == 1 and msg.endswith("bm25x_lookup_terms: index was created without term keys")


def test_device_refusals_leave_no_memory(m):
    bm = _bm(m)
    zero = write_tsvectors([[(b"ok", [1])], [(b"a", [1]), (b"nopos", [])]])     # haspos with 0 positions: count 0
    flat, off = word_table([b"many"])
    # 257 entries of one lexeme, all pointing at the same 65535 positions: merged tf 257 * 65535 >= 2^24
    big = pack_ids([1], flat, off, np.zeros(1, np.int64), [65535])
    big["entries"] = np.repeat(big["entries"], 257)
    big["ent_off"] = np.array([0, 257], np.uint64)
    ix0 = m.Index.from_tsvectors(SEED, **pack_sorted([{b"warm": [1]}]))        # CUDA context and pools warmed up
    ix0.tsvector_queries(SEED, **pack_sorted([{b"warm": [1]}]))
    before = free_bytes()
    for as_query in (False,):
        code, msg = refused(m, lambda: bm.cast_tsvectors(SEED, **zero, as_query=as_query))
        assert (code, msg) == (1, "bm25x error 1: bm25x_cast_tsvectors: invalid data: a lexeme of tsvector 1 has "
                                  "position counts that sum to 0")
    assert bm.cast_tsvectors(SEED, **zero, as_query=True)[0].tolist() == [0, 1, 3]
    code, msg = refused(m, lambda: m.Index.from_tsvectors(SEED, **zero))
    assert code == 1 and "bm25x_index_create_from_tsvectors: invalid data: a lexeme of tsvector 1" in msg
    off, keys, tf = bm.cast_tsvectors(SEED, **big)
    assert tf.tolist() == [257 * 65535]
    code, msg = refused(m, lambda: m.Index.from_tsvectors(SEED, **big))
    assert (code, msg) == (4, "bm25x error 4: bm25x_index_create_from_tsvectors: term frequency >= 2^24 is not "
                              "supported by the packed posting layout (document 0)")
    code, msg = refused(m, lambda: m.Index.from_tsvectors(SEED, **pack_sorted([{b"a": [1]}]), device=99))
    assert code == 2 and "bm25x_index_create_from_tsvectors: CUDA device 99 not available" in msg
    assert free_bytes() == before
