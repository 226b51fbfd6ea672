"""GPU: document ids across the whole 32-bit range, up to the largest the library accepts (n_docs = 2^32 - 2, ids up to
0xFFFFFFFD; 0xFFFFFFFF is the pad slot, the exhausted cursor and the empty result slot at once).

A few hundred thousand postings placed on purpose (tests/util_sparse.py: high_id_corpus) — around 2^31, near 3 * 2^30,
in the top 2048 ids, tie groups on both sides of 2^31, pad slots after the last id, a bit-width-32 block and a
byte-width-4 tail above 2^31 — in indexes of ~2^32 documents, checked bit for bit against the sparse exact reference of
tests/util_sparse.py (pinned against the oracle by tests/test_sparse_reference.py): the device arrays, every kernel path
with pruning on and off, the prefilter bitmap, the HBM candidate pools, a growing segment whose ids end at 0xFFFFFFFD,
and a document-sharded index with shard bounds at 2^31 and next to the last id.

Each index holds ~7 bytes per document on the device (fieldnorm, payload): ~30 GB.  One is alive at a time; building
one takes ~34 GB of host memory (the norms and the synthesised payload) and ~47 GB through the CSR path (plus 4-byte
lengths), as measured on an H100 host; the sharded index builds one shard at a time.  Each build is skipped, saying so,
when the free device or available host memory is short of that."""
import ctypes
import time
from types import SimpleNamespace

import numpy as np
import pytest

import _pkg
from util_cuda import cudart, download
from util_index import LAYOUT, ctid
from util_sparse import (DOC_INF, FN_EMPTY, FN_TIE, MAX_N_DOCS, T31, SparseReference, assert_rows, full_fieldnorm,
                         high_id_corpus, reference, sum_len_of)

pytestmark = pytest.mark.gpu

N_A = MAX_N_DOCS - 64       # index A: room for a growing segment of 64 documents, ids up to 0xFFFFFFFD
N_B = MAX_N_DOCS            # sharded index B: the largest n_docs
K1, B = 1.2, 0.75
KS = (1, 10, 128, 129, 224, 1025)
# kernel paths of the 2..8-term classes (test_gpu_paths.PATHS and the hand-back / dense options of
# test_gpu_parity.test_kernel_paths_identical): (seed, twophase, seed_prune_min, seed_dense_div)
PATHS = dict(seeded=(1, 0, 0xFFFFFFFF, 0), handback=(1, 0, 64, 0), dense=(1, 0, 0xFFFFFFFF, 8), twophase=(0, 1, 0, 0),
             plain=(0, 0, 0, 0))


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


def _need(host_gb, dev_gb, what):
    import psutil
    free, total = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert cudart().cudaMemGetInfo(ctypes.byref(free), ctypes.byref(total)) == 0
    host = psutil.virtual_memory().available
    if host < host_gb * 1e9 or free.value < dev_gb * 1e9:
        pytest.skip(f"{what} needs {host_gb} GB of host and {dev_gb} GB of free device memory "
                    f"({host / 1e9:.0f} GB / {free.value / 1e9:.0f} GB available)")


def _peak_host_gb():
    import resource
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6


_alive = {}  # the one large index alive at a time


def _build(name, make):
    for h in _alive.values():
        h.close()
    _alive.clear()
    t0 = time.perf_counter()
    ix = make()
    print(f"\n[high-id] {name}: built in {time.perf_counter() - t0:.1f} s, "
          f"{ix.info().device_bytes / 1e9:.1f} GB on the device, host peak so far {_peak_host_gb():.1f} GB")
    _alive[name] = ix
    return ix


@pytest.fixture(scope="module", autouse=True)
def _close_last():
    t0 = time.perf_counter()
    yield
    for h in _alive.values():
        h.close()
    _alive.clear()
    print(f"\n[high-id] module wall time {time.perf_counter() - t0:.0f} s, host peak {_peak_host_gb():.1f} GB")


@pytest.fixture(scope="module")
def corpus_a(orc):
    c = high_id_corpus(N_A)
    return c, reference(orc, c, K1, B)


@pytest.fixture(scope="module")
def encoded_a(orc, corpus_a):
    c, _ = corpus_a
    return orc.EncodedBlocks(SimpleNamespace(n_terms=c.n_terms, post_off=c.post_off, post_doc=c.post_doc,
                                             post_tf=c.post_tf))


@pytest.fixture(scope="module")
def index_a(m, orc, corpus_a, encoded_a):
    """Index A from the stored blocks (norms + sum of lengths, as the pages hold them)."""
    c, _ = corpus_a
    eb = encoded_a
    _need(45, 34, "index A (2^32 - 66 documents)")

    def make():
        fn = full_fieldnorm(c)
        return m.Index.from_blocks(c.n_docs, c.n_terms, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf,
                                   eb.doc_off, eb.tf_off, eb.bytes[:eb.n_bytes], doc_fieldnorm=fn,
                                   sum_doc_len=sum_len_of(orc, c), k1=K1, b=B)
    return _build("index A from blocks", make)


def _queries(c, seed):
    """Queries of 1, 2, 3, 4, 5-8, 9-16, 17-32 and 33-64 live terms over the corpus' kinds of terms."""
    k = c.kinds
    rng = np.random.default_rng(seed)
    rand = lambda n: rng.choice(c.n_terms, n, replace=False)
    qs = [[t] for t in k["tie"] + k["dense"][:2] + k["pad"] + k["wide"] + k["head"][:1] + k["fill"][-2:]]
    qs += [[k["tie"][0], k["dense"][0]], [k["head"][0], k["tie"][1]], k["dense"][:2], [k["pad"][0], k["tie"][2]]]
    qs += [k["dense"][:3], [k["head"][0], k["head"][1], k["tie"][0]], k["tie"]]
    qs += [k["dense"][:4], k["pad"] + k["dense"][:2] + k["wide"], k["tie"] + k["pad"]]
    qs += [k["dense"] + k["pad"], k["head"] + k["tie"], list(rand(5)), list(rand(8))]
    qs += [k["dense"] + k["tie"] + list(rand(3)), list(rand(16)), list(rand(17)), list(rand(32)), list(rand(33)),
           list(rand(64))]
    qs = [np.unique(np.asarray(q, np.uint32)) for q in qs]
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    return q_off, np.concatenate(qs).astype(np.uint32), qs


class _Prefix:
    """SparseReference.search at one limit per (query, bitmap): every smaller limit's rows are a prefix."""

    def __init__(self, ref, kmax):
        self.ref, self.kmax, self.memo = ref, kmax, {}

    def search(self, terms, k, allow=None):
        key = (np.asarray(terms, np.uint32).tobytes(), id(allow))
        if key not in self.memo:
            self.memo[key] = self.ref.search(terms, self.kmax, allow=allow)
        r = self.memo[key]
        n = min(k, r.n)
        return SimpleNamespace(doc=r.doc[:n], score64=r.score64[:n], score=r.score[:n], payload=r.payload[:n], n=n)


def _set_path(ix, name):
    seed, two, spm, div = PATHS[name]
    ix.set_option("seed", seed)
    ix.set_option("twophase", two)
    ix.set_option("seed_prune_min", spm)
    ix.set_option("seed_dense_div", div)


def _rows_identical(a, b, what):
    for key in ("doc", "score", "score64", "n", "payload"):
        assert np.array_equal(a[key], b[key]), f"{what}: {key}"


def _slices(n):
    """First 4 KiB, the 4 KiB around 2^31 and the last 4 KiB of the doc ids [0, n)."""
    return [(0, 4096), (T31 - 2048, T31 + 2048), (n - 4096, n)]


def _check_arrays(ix, ref, c, what):
    lay, der = ix.layout(), ix.derived()
    r = ref.arrays()
    for name in ("n_docs", "n_terms", "n_postings", "n_postings_padded", "n_blocks", "sum_doc_len", "k1", "b", "avgdl"):
        assert getattr(lay, name) == getattr(r, name), f"{what}: layout.{name} {getattr(lay, name)} != {getattr(r, name)}"
    assert der.n_champ == r.n_champ and der.s1f_min == r.s1f_min, what
    got = {}
    for i, (name, dt) in enumerate(LAYOUT):
        if name not in ("fieldnorm", "payload"):
            got[name] = download(lay.dev_ptr[i], lay.bytes[i], dt)
    for name, dt in (("pdoc", np.uint32), ("champ", np.uint32), ("champ_off", np.uint64)):
        got[name] = download(getattr(der, name), getattr(der, name + "_bytes"), dt)
    for name, have in got.items():
        want = getattr(r, name)
        assert have.shape == want.shape, f"{what}: {name} {have.shape} != {want.shape}"
        if not np.array_equal(have, want):
            bad = np.flatnonzero(have != want)
            raise AssertionError(f"{what}: {name} differs at {len(bad)} entries, first {bad[:4].tolist()}: "
                                 f"device {have[bad[:4]].tolist()} reference {want[bad[:4]].tolist()}")
    # the largest id is followed by pad slots, then the slack
    (p,) = c.kinds["pad"]
    end = int(r.post_off[p]) + int(r.df[p])
    assert got["post"][2 * (end - 1)] == c.n_docs - 1 and got["post"][2 * end] == DOC_INF
    # per-document arrays on slices: norms and the synthetic ctid of every id
    fi, pi = [n for n, _ in LAYOUT].index("fieldnorm"), [n for n, _ in LAYOUT].index("payload")
    assert lay.bytes[fi] == c.n_docs and lay.bytes[pi] == 6 * c.n_docs
    for lo, hi in _slices(c.n_docs):
        fn = download(lay.dev_ptr[fi] + lo, hi - lo, np.uint8)
        want = np.full(hi - lo, FN_EMPTY, np.uint8)
        sel = (c.live >= lo) & (c.live < hi)
        want[c.live[sel] - lo] = c.live_fn[sel]
        assert np.array_equal(fn, want), f"{what}: fieldnorm [{lo}, {hi})"
        pl = download(lay.dev_ptr[pi] + 6 * lo, 6 * (hi - lo), np.uint16).reshape(-1, 3)
        assert np.array_equal(pl, ctid(np.arange(lo, hi))), f"{what}: payload [{lo}, {hi})"


def test_index_a_arrays(index_a, corpus_a):
    c, ref = corpus_a
    _check_arrays(index_a, ref, c, "index A (blocks)")


def test_stored_blocks_above_2_31(index_a, corpus_a, encoded_a):
    """The wide term is stored as a bit-width-32 full block (raw ids, bitpacking_u32_ordered.rs:119-121) and a
    byte-width-4 tail (raw ids, bytepacking_u32_ordered.rs:195,211) above 2^31; decoded on the GPU to its ids."""
    c, ref = corpus_a
    eb = encoded_a
    (w,) = c.kinds["wide"]
    g = int(eb.term_blk_off[w])
    assert int(eb.term_blk_off[w + 1]) == g + 2 and eb.meta_doc[g] == 32 and eb.meta_doc[g + 1] == 0x80 | 4
    ids = c.post_doc[int(c.post_off[w]):int(c.post_off[w + 1])]
    assert ids[128] >= T31
    got = index_a.search_batch(np.array([0, 1], np.uint32), np.array([w], np.uint32), 1025, want_payload=True)
    assert sorted(got["doc"][0, :int(got["n"][0])].tolist()) == ids.tolist()
    assert_rows(got, ref, [[w]], 1025, "wide term")


def test_index_a_kernel_paths(index_a, corpus_a):
    """Every kernel path with pruning on and off: the same rows, equal to the sparse reference (ids, f64 and f32
    scores, payload, empty slots)."""
    c, ref = corpus_a
    ix = index_a
    q_off, q_terms, qs = _queries(c, 11)
    pref = _Prefix(ref, max(KS))
    for k in KS:
        got = {}
        for name in PATHS:
            for prune in (1, 0):
                _set_path(ix, name)
                ix.set_option("prune", prune)
                got[name, prune] = ix.search_batch(q_off, q_terms, k, want_payload=True)
                assert got[name, prune]["stats"].launches >= 1
        for key, res in got.items():
            _rows_identical(res, got["plain", 1], f"{key} k={k}")
        assert_rows(got["seeded", 1], pref, qs, k, f"paths k={k}")
    _set_path(ix, "seeded")
    ix.set_option("seed_prune_min", 32768)
    ix.set_option("seed_dense_div", 64)
    ix.set_option("prune", 1)


def test_index_a_prefilter(index_a, corpus_a):
    """Bitmaps over 2^32 - 66 documents (512 MiB): bits set and cleared at 2^31 - 1 and 2^31, in the last partial byte
    and at the last document."""
    c, ref = corpus_a
    ix = index_a
    rng = np.random.default_rng(5)
    q_off, q_terms, qs = _queries(c, 12)
    nbytes = (c.n_docs + 7) // 8
    assert c.n_docs % 8 != 0
    for flip in (0, 1):
        allow = np.zeros(nbytes, np.uint8)
        on = c.live[rng.random(len(c.live)) < 0.5]
        np.bitwise_or.at(allow, on >> 3, (1 << (on & 7)).astype(np.uint8))
        for d, bit in ((T31 - 1, 1 - flip), (T31, flip), (c.n_docs - 1, 1 - flip), (c.n_docs - 3, flip)):
            if bit:
                allow[d >> 3] |= np.uint8(1 << (d & 7))
            else:
                allow[d >> 3] &= np.uint8(~(1 << (d & 7)) & 0xFF)
        pref = _Prefix(ref, 1025)
        for k in (10, 129, 1025):
            for prune in (1, 0):
                ix.set_option("prune", prune)
                res = ix.search_batch(q_off, q_terms, k, allow=allow, want_payload=True)
                assert_rows(res, pref, qs, k, f"prefilter flip={flip} k={k} prune={prune}", allow=allow)
    ix.set_option("prune", 1)


def test_index_a_hbm_pools(index_a, corpus_a):
    """Limits 1025 and 65 535 (candidate pools in HBM) on queries matching more than 65 535 documents."""
    c, ref = corpus_a
    head = c.kinds["head"]
    qs = [np.array(head[:3], np.uint32), np.array(head, np.uint32), np.array(head[:2] + c.kinds["tie"], np.uint32)]
    q_off = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint32)
    q_terms = np.concatenate(qs)
    pref = _Prefix(ref, 65535)
    assert pref.search(qs[0], 65535).n == 65535
    for k in (1025, 65535):
        for prune in (1, 0):
            index_a.set_option("prune", prune)
            res = index_a.search_batch(q_off, q_terms, k, want_payload=True)
            assert_rows(res, pref, qs, k, f"hbm pool k={k} prune={prune}")
    index_a.set_option("prune", 1)


def _growing_docs(c, G, seed):
    """G growing documents over the corpus' tie, pad and dense terms; the last one the best match of the pad term."""
    rng = np.random.default_rng(seed)
    pool = c.kinds["tie"] + c.kinds["pad"] + c.kinds["dense"][:2]
    elems = []
    for g in range(G):
        t = np.sort(rng.choice(pool, int(rng.integers(1, 4)), replace=False))
        tf = np.ones(len(t), np.uint32) if g % 3 == 0 else rng.integers(1, 5, len(t)).astype(np.uint32)
        elems.append((t, tf))
    elems[-1] = (np.array(c.kinds["pad"], np.int64), np.array([40], np.uint32))
    off = np.cumsum([0] + [len(t) for t, _ in elems]).astype(np.uint64)
    fn = np.where(np.arange(G) % 3 == 0, FN_TIE, 30).astype(np.uint8)   # tf 1 at FN_TIE ties with sealed documents
    return off, np.concatenate([t for t, _ in elems]).astype(np.uint32), np.concatenate([f for _, f in elems]), fn


def test_index_a_growing_ids_up_to_the_last(m, orc, index_a, corpus_a):
    """Sealed n_docs + 64 growing documents = 2^32 - 2: merged ids run up to 0xFFFFFFFD and equal the reference over
    sealed + growing scored with the sealed statistics.  One more growing document is refused."""
    c, ref = corpus_a
    G = 64
    off, term, tf, gfn = _growing_docs(c, G, 21)
    gix = index_a.growing(off, term, tf, doc_fieldnorm=gfn)
    # the reference over both: each term's sealed list, then its growing documents at n_docs + ordinal
    gdoc = np.repeat(np.arange(G), np.diff(off.astype(np.int64)))
    lists_doc, lists_tf, lists_fn = [], [], []
    for t in range(c.n_terms):
        s0, s1 = int(c.post_off[t]), int(c.post_off[t + 1])
        sel = term == t
        lists_doc.append(np.concatenate([c.post_doc[s0:s1].astype(np.int64), N_A + gdoc[sel]]))
        lists_tf.append(np.concatenate([c.post_tf[s0:s1], tf[sel]]))
        lists_fn.append(np.concatenate([ref.post_fn[s0:s1], gfn[gdoc[sel]]]))
    both_off = np.concatenate([[0], np.cumsum([len(d) for d in lists_doc])])
    both = SparseReference(orc, N_A + G, both_off, np.concatenate(lists_doc), np.concatenate(lists_tf), K1, B, ref.sum_len,
                           post_fn=np.concatenate(lists_fn), norms=ref.norms, stat=(N_A, ref.df, ref.sum_len / N_A))
    q_off, q_terms, qs = _queries(c, 13)
    pref = _Prefix(both, 1025)
    top = 0
    for k in (1, 10, 129, 1025):
        res = index_a.search_batch_growing(gix, q_off, q_terms, k, want_payload=True)
        assert_rows(res, pref, qs, k, f"sealed + growing k={k}",
                    payload_of=lambda d: ctid(np.where(d >= N_A, d.astype(np.int64) - N_A, d)))
        top = max(top, int(res["doc"][res["doc"] != DOC_INF].max()))
    assert top == MAX_N_DOCS - 1 == 0xFFFFFFFD
    gix.close()
    off, term, tf, gfn = _growing_docs(c, G + 1, 22)
    with pytest.raises(m.Bm25xError, match=f"{N_A}.*{G + 1}") as e:
        index_a.growing(off, term, tf, doc_fieldnorm=gfn)
    assert e.value.code == 1


def test_index_a_again_from_the_csr(m, orc, index_a, corpus_a):
    """The same index through bm25x_index_create (exact lengths, k_build_postings), after index A is closed: the same
    bits."""
    c, ref = corpus_a
    index_a.close()
    _need(60, 34, "index A from the CSR (4-byte lengths of 2^32 - 66 documents)")
    L = orc.lib()
    length = np.array([L.orc_fieldnorm_to_length(f) for f in range(256)], dtype=np.uint32)

    def make():
        doc_len = np.full(c.n_docs, length[FN_EMPTY], np.uint32)
        doc_len[c.live] = length[c.live_fn]
        return m.Index(c.n_docs, doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=K1, b=B)
    ix = _build("index A from the CSR", make)
    _check_arrays(ix, ref, c, "index A (CSR)")
    ix.close()


def test_sharded_index_b(m, orc):
    """ShardedIndex over n_docs = 2^32 - 2 with shard bounds [0, 2^31, 2^31 + 3, N - 5, N] (shards of 3 and 5
    documents, bounds that are not multiples of 8 at high offsets): every output row equals the reference over global
    ids (payload = ctid of the global id), with and without a prefilter bitmap, at limits of every pool class.  (The
    balanced default bounds take an 8-byte prefix sum per document, 34 GB here: bm25x_sharded_create's default bounds are
    tested at smaller sizes by tests/test_gpu_sharded.py.)"""
    _need(45, 34, "sharded index B (2^32 - 2 documents)")
    c = high_id_corpus(N_B)
    ref = reference(orc, c, K1, B)
    L = orc.lib()
    length = np.array([L.orc_fieldnorm_to_length(f) for f in range(256)], dtype=np.uint32)
    S, doc_bounds = 4, np.array([0, T31, T31 + 3, N_B - 5, N_B], np.uint32)

    def make():
        doc_len = np.full(c.n_docs, length[FN_EMPTY], np.uint32)
        doc_len[c.live] = length[c.live_fn]
        return m.ShardedIndex(c.n_docs, doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=K1, b=B, n_shards=S,
                              doc_bounds=doc_bounds)
    sx = _build("sharded index B", make)
    assert np.array_equal(sx.doc_bounds(), doc_bounds)
    q_off, q_terms, qs = _queries(c, 14)
    rng = np.random.default_rng(6)
    allow = np.zeros((N_B + 7) // 8, np.uint8)
    on = c.live[rng.random(len(c.live)) < 0.5]
    np.bitwise_or.at(allow, on >> 3, (1 << (on & 7)).astype(np.uint8))
    allow[(T31 + 2) >> 3] |= np.uint8(1 << ((T31 + 2) & 7))
    for al in (None, allow):
        pref = _Prefix(ref, 1025)
        for k in (1, 10, 129, 1025):
            res = sx.search_batch(q_off, q_terms, k, allow=al, want_payload=True)
            assert_rows(res, pref, qs, k, f"sharded k={k} allow={al is not None}", allow=al)
    sx.close()
    _alive.clear()
