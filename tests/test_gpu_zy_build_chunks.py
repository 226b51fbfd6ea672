"""The builds from documents and tsvectors at the sizes only a large batch reaches: a keyed corpus of 4.2 chunks whose
vocabulary pass regrows keeping 8.3 M entries, defers a compaction and then compacts two appended chunks at once; and a
batch of 3 * 2^22 + 2^20 tsvectors cut by the vector count (the widest vector bits of the cast's sort, a chunk of empty
vectors), cast, built, turned into queries and inserted into a growing segment of more than 2^22 rows.

Each fixture's CPU test asserts on the restated schedules (util_documents.vocab_schedule, util_tsvector.cast_cuts) that
it reaches its branches.  The GPU tests compare with the Segment restatement built by the CSR build, the oracle, the host
cast over bm25x_intern and, for the growing segment, its twin fed the restated rows."""
import numpy as np
import pytest

from util_cuda import download
from util_documents import CHUNK, csr_kwargs, segment, vocab_schedule
from util_growing_tsvector import SEED, Twin, bm_of, same_seal, same_segment
from util_index import DERIVED, LAYOUT, SCALARS, read_back
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import PrefixOracle, compare, oracle_index, query_csr, same_rows
from util_sparse import need
from util_tsvector import CHUNK_VEC, byte_cut_batch, cast, cast_cuts, pack_ids, pack_sorted, word_table

SLICE = 1 << 28


# ---- a: 4.2 chunks of keyed documents over 17.4 M distinct keys ----

N_A, L_A = 176_000, 100
SHARED_HI = 1 << 63        # the key of every document: (2^63, 0), big-endian words


def _large_corpus():
    """N_A documents of L_A keys: 99 random ones (distinct with overwhelming odds) and the shared key, ascending."""
    rng = np.random.default_rng(0xA4)
    hi = rng.integers(0, 1 << 63, (N_A, L_A), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, (N_A, L_A),
                                                                                            dtype=np.uint64)
    lo = rng.integers(0, 1 << 63, (N_A, L_A), dtype=np.uint64)
    hi[:, 0], lo[:, 0] = SHARED_HI, 0
    order = np.argsort(hi, axis=1, kind="stable")
    hi, lo = np.take_along_axis(hi, order, 1), np.take_along_axis(lo, order, 1)
    assert (np.diff(hi, axis=1) > 0).all()
    words = np.empty((N_A * L_A, 2), ">u8")
    words[:, 0], words[:, 1] = hi.reshape(-1), lo.reshape(-1)
    del hi, lo, order
    off = np.arange(N_A + 1, dtype=np.uint64) * np.uint64(L_A)
    tf = rng.integers(1, 20, N_A * L_A).astype(np.uint32)
    return dict(elem_off=off, elem_tf=tf, elem_key=words.view(np.uint8).reshape(-1, 16))


@pytest.fixture(scope="module")
def large():
    return _large_corpus()


def test_large_corpus_regrows_defers_and_compacts_two_chunks(large):
    E = len(large["elem_key"])
    assert 4 * CHUNK < E < 5 * CHUNK
    ev = vocab_schedule(large["elem_key"])
    kinds = [(e[0], e[1]) for e in ev]
    assert kinds == [("grow", 0), ("compact", 0), ("compact", 1), ("grow", 2), ("defer", 2), ("compact", 3),
                     ("compact", 4)], ev
    assert ev[0][3] == 0
    assert ev[3][3] > 8_000_000                                     # the regrow keeps the compacted list
    assert ev[4][2] == CHUNK and ev[5][2] == 2 * CHUNK              # deferred, then two appended chunks compacted


def _same_device_bytes(a_ptr, b_ptr, nbytes, what):
    for o in range(0, int(nbytes), SLICE):
        n = min(SLICE, int(nbytes) - o)
        assert download(a_ptr + o, n, np.uint8).tobytes() == download(b_ptr + o, n, np.uint8).tobytes(), f"{what} @ {o}"


@pytest.mark.gpu
def test_large_keyed_corpus_equals_the_segment_build(m, orc, large):
    need(24, 16, "17.6 M keyed elements beside their Segment")
    s = segment(large["elem_off"], large["elem_tf"], elem_key=large["elem_key"])
    got = m.Index.from_documents(**large)
    want = m.Index(**csr_kwargs(s))
    lg, lw = got.layout(), want.layout()
    for name in SCALARS:
        assert getattr(lg, name) == getattr(lw, name), name
    for i, (name, _) in enumerate(LAYOUT):
        assert lg.bytes[i] == lw.bytes[i], name
        _same_device_bytes(lg.dev_ptr[i], lw.dev_ptr[i], lw.bytes[i], name)
    dg, dw = got.derived(), want.derived()
    assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min
    for name in ("pdoc", "champ", "champ_off"):
        assert getattr(dg, name + "_bytes") == getattr(dw, name + "_bytes"), name
        _same_device_bytes(getattr(dg, name), getattr(dw, name), getattr(dw, name + "_bytes"), name)
    assert np.array_equal(got.df(), want.df())
    a, w = got.info(), want.info()
    assert [getattr(a, f) for f, _ in type(a)._fields_] == [getattr(w, f) for f, _ in type(w)._fields_]
    assert np.array_equal(got.lookup_terms(s.term_keys), np.arange(s.n_terms, dtype=np.uint32))
    # queries: the shared key with keys of documents across the chunks
    shared_key = np.zeros((1, 16), np.uint8)
    shared_key[0, 0] = 0x80                                         # (SHARED_HI, 0) as bytes
    shared = int(got.lookup_terms(shared_key)[0])
    assert s.post_off[shared + 1] - s.post_off[shared] == N_A
    rng = np.random.default_rng(4)
    qs = []
    for i in range(240):
        at = rng.integers(0, N_A * L_A, int(rng.integers(1, 6)))   # keys of elements across every chunk
        q = set(got.lookup_terms(large["elem_key"][at]).tolist())
        if i % 3:
            q.add(shared)
        qs.append(sorted(q))
    q_off, q_terms = query_csr(qs)
    oix = PrefixOracle(oracle_index(orc, s), 1000)
    for k in (1, 10, 100, 1000):
        r = got.search_batch(q_off, q_terms, k, want_payload=True)
        same_rows(r, want.search_batch(q_off, q_terms, k, want_payload=True), f"k={k}")
        compare(r, oix, q_off, q_terms, k, what=f"oracle k={k}")


# ---- f: 3 * 2^22 + 2^20 tsvectors, cut by the vector count ----

N_F = 3 * CHUNK_VEC + (1 << 20)
EDGE_F = (0, CHUNK_VEC - 1, CHUNK_VEC)      # vectors that share the key of b"shared"


def _words_f():
    rng = np.random.default_rng(0xF0)
    words = list(dict.fromkeys(bytes(rng.integers(97, 123, int(rng.integers(3, 11)), dtype=np.uint8))
                               for _ in range(2500)))
    return [b"shared"] + [w for w in words if w != b"shared"][:2000]


def _vector_batch(words, fresh_from=None):
    """N_F tsvectors, one in 64 non-empty over [0, 2^23) and one in 4096 over [3 * 2^22, N_F), the rest (the whole of
    [2^23, 3 * 2^22) among them) empty; vectors EDGE_F hold b"shared".  Entries are words[1:fresh_from] except in the
    vectors below 2^16 and from 3 * 2^22 on, which draw from all the words (fresh_from: the first word the sealed side
    lacks).  Returns (tsv, word id per entry)."""
    rng = np.random.default_rng(0xF1)
    live = np.concatenate([np.arange(5, 2 * CHUNK_VEC, 64), np.arange(3 * CHUNK_VEC + 7, N_F, 4096), EDGE_F])
    live = np.unique(live)
    lens = np.zeros(N_F, np.int64)
    lens[live] = rng.integers(1, 7, len(live))
    vec = np.repeat(np.arange(N_F), lens)
    hi = np.where((vec < (1 << 16)) | (vec >= 3 * CHUNK_VEC), len(words), fresh_from or len(words))
    wid = 1 + (rng.random(len(vec)) * (hi - 1)).astype(np.int64)
    # distinct words within a vector: keep the first of each (vector, word), then put b"shared" first in EDGE_F
    pair = vec * len(words) + wid
    _, keep = np.unique(pair, return_index=True)
    keep.sort()
    vec, wid = vec[keep], wid[keep]
    for v in EDGE_F:
        wid[np.searchsorted(vec, v)] = 0
    lens = np.bincount(vec, minlength=N_F)
    flat, off = word_table(words)
    return pack_ids(lens, flat, off, wid, rng.integers(1, 5, len(wid))), wid


@pytest.fixture(scope="module")
def vectors():
    return _vector_batch(_words_f())[0]


def test_vector_batch_cuts_on_vector_count(vectors):
    cuts = cast_cuts(vectors)
    V = CHUNK_VEC
    assert [(a, b, r) for a, b, r, _ in cuts] == [(0, V, "vectors"), (V, 2 * V, "vectors"), (2 * V, 3 * V, "vectors"),
                                                 (3 * V, N_F, "end")]
    assert cuts[2][3] == 0 and all(c[3] > 0 for i, c in enumerate(cuts) if i != 2)   # chunk 2: ne == 0, skipped
    # the vectors of EDGE_F share a key: the first and last of chunk 0 (sorted over 22 vector bits), the first of chunk 1
    off, keys, _ = cast(None, SEED, vectors, keys=_keys_f(vectors))
    for v in EDGE_F:
        assert b"shared" in {bytes(k).rstrip(b"\0") for k in keys[int(off[v]):int(off[v + 1])]}


def _keys_f(tsv):
    """Keys of the batch's lexemes (short, NUL-free): zero-padded (the copy path)."""
    ent_off = np.asarray(tsv["ent_off"], np.int64)
    e = np.asarray(tsv["entries"], np.uint32).astype(np.int64)
    vec = np.repeat(np.arange(len(ent_off) - 1), np.diff(ent_off))
    start = np.asarray(tsv["byte_off"], np.int64)[:-1][vec] + (e >> 12)
    ln = (e >> 1) & 0x7FF
    assert (ln < 16).all()
    j = np.arange(15)
    mask = j[None, :] < ln[:, None]
    keys = np.zeros((len(e), 16), np.uint8)
    keys[:, :15] = np.where(mask, np.asarray(tsv["data"])[np.where(mask, start[:, None] + j[None, :], 0)], 0)
    return keys


def _same_arrays(lg, dg, lw, dw, what):
    for name in SCALARS:
        assert getattr(lg, name) == getattr(lw, name), f"{what}: {name}"
    assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min, what
    ag, aw = read_back(lg, dg), read_back(lw, dw)
    for name, _ in LAYOUT + DERIVED:
        if (name in ("blk", "blk_ub") and lw.n_blocks == 0) or (name == "champ" and dw.n_champ == 0):
            continue
        assert ag[name].tobytes() == aw[name].tobytes(), f"{what}: {name} differs"


@pytest.mark.gpu
def test_vector_batch_cast_build_and_queries(m, orc, vectors):
    need(16, 8, "3 * 2^22 + 2^20 tsvectors")
    bm = bm_of(m)
    keys = _keys_f(vectors)
    for as_query in (False, True):
        got = bm.cast_tsvectors(SEED, **vectors, as_query=as_query)
        want = cast(bm.intern, SEED, vectors, as_query=as_query, keys=keys)
        assert np.array_equal(got[0], want[0]), f"query={as_query}: offsets"
        assert got[1].tobytes() == want[1].tobytes(), f"query={as_query}: keys"
        assert as_query or np.array_equal(got[2], want[2]), "tf"
    off = got[0]
    assert (off[2 * CHUNK_VEC:3 * CHUNK_VEC + 1] == off[2 * CHUNK_VEC]).all()    # the empty chunk: rows of 0
    c_off, c_keys, c_tf = cast(bm.intern, SEED, vectors, keys=keys)
    s = segment(c_off, c_tf, elem_key=c_keys)
    ix = m.Index.from_tsvectors(SEED, **vectors)
    csr = m.Index(**csr_kwargs(s))
    _same_arrays(ix.layout(), ix.derived(), csr.layout(), csr.derived(), "vectors")
    a, w = ix.info(), csr.info()
    assert [getattr(a, f) for f, _ in type(a)._fields_] == [getattr(w, f) for f, _ in type(w)._fields_]
    q_off, q_terms = ix.tsvector_queries(SEED, **vectors)
    qo, qk, _ = cast(bm.intern, SEED, vectors, as_query=True, keys=keys)
    assert np.array_equal(q_off, qo.astype(np.uint32)) and np.array_equal(q_terms, csr.lookup_terms(qk))
    rows = np.flatnonzero(np.diff(q_off.astype(np.int64)))
    pick = np.unique(np.concatenate([np.arange(0, len(rows), len(rows) // 150), np.searchsorted(rows, EDGE_F)]))
    p_off, p_terms = query_csr([q_terms[q_off[rows[i]]:q_off[rows[i] + 1]] for i in pick])
    oix = PrefixOracle(oracle_index(orc, s), 1000)
    for k in (1, 10, 100, 1000):
        r = ix.search_batch(p_off, p_terms, k, want_payload=True)
        same_rows(r, csr.search_batch(p_off, p_terms, k, want_payload=True), f"k={k}")
        compare(r, oix, p_off, p_terms, k, what=f"oracle k={k}")


# ---- the growing segment's tsvector insert of batches f and e ----

def _sealed(m, kind, words):
    """A keyed sealed side of 3 000 documents over words."""
    rng = np.random.default_rng(len(words))
    docs = [{words[int(w)]: [1, 2][:int(rng.integers(1, 3))] for w in rng.choice(len(words), int(rng.integers(1, 12)),
                                                                               replace=False)} for _ in range(3000)]
    tsv = pack_sorted(docs)
    if kind == "index":
        return m.Index.from_tsvectors(SEED, **tsv)
    off, keys, tf = cast(bm_of(m).intern, SEED, tsv)
    return m.ShardedIndex.from_documents(off, tf, elem_key=keys, n_shards=2)


def test_growing_batch_has_fresh_keys_at_both_ends():
    words = _words_f()
    tsv, wid = _vector_batch(words, fresh_from=1500)
    vec = np.repeat(np.arange(N_F), np.diff(tsv["ent_off"].astype(np.int64)))
    fresh = vec[wid >= 1500]
    assert len(fresh) and fresh.max() >= 3 * CHUNK_VEC and fresh.min() < 1 << 16
    assert not ((fresh >= 1 << 16) & (fresh < 3 * CHUNK_VEC)).any()
    assert N_F > 1 << 22                                            # the segmented sort's rows: more than 2^22


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["index", "sharded2"])
def test_growing_insert_of_the_cut_batches_equals_twin(m, orc, kind):
    need(24, 8, "a growing segment of 3 * 2^22 + 2^20 tsvectors")
    words = _words_f()
    sealed = _sealed(m, kind, words[:1500])
    seg, twin = sealed.growing_segment(), Twin(m, sealed)
    f, _ = _vector_batch(words, fresh_from=1500)
    seg.insert_tsvectors(SEED, **f)
    twin.insert(orc, f)
    assert len(twin.keys) > 0
    rng = np.random.default_rng(6)
    q = pack_sorted([{words[int(w)]: [1] for w in rng.integers(0, len(words), int(rng.integers(1, 6)))}
                     for _ in range(60)])
    same_segment(seg, twin, q, f"{kind} vectors")
    e, long_words, _ = byte_cut_batch(seed=23)
    seg.insert_tsvectors(SEED, **e)
    twin.insert(orc, e)
    q2 = pack_sorted([{long_words[int(w)]: [1] for w in rng.integers(0, len(long_words), 3)} for _ in range(40)])
    same_segment(seg, twin, q2, f"{kind} bytes")
    same_seal(seg.seal(), twin.seg.seal(new_keys=twin.new_keys()), f"{kind} seal")
