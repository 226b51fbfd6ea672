"""GPU: every array of every kind of index handle against the CPU restatement of tests/util_index.py, bit for bit — the 13
arrays of bm25x_index_layout and the derived ones no search row shows directly: the doc-id copy the seeded rings stream
(pad and slack slots 0xFFFFFFFF) and the champion lists the seeded kernel takes its single-term documents from
(k_champions: one warp per term, a 256-entry buffer behind a running threshold, cut back to 128 by a bitonic sort).

Handles: bm25x_index_create (synthetic shapes and a champion edge corpus), stored-block ingest (both norm forms), a
replica finalized twice, a growing segment (sealed statistics), and every shard of a document-sharded index (local ids,
the whole segment's statistics)."""
import numpy as np
import pytest

import _pkg
from util_cuda import D2D, cudart, sm_count
from util_index import (CHAMP_L, assert_matches, cache, champion_lists, fieldnorms, read_back, restate)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


def _check(ix, r, what, skip=()):
    lay, der = ix.layout(), ix.derived()
    got = read_back(lay, der)
    assert_matches(got, lay, der, r, what, skip)
    return got


def _csr(lists):
    """Term-major CSR (off, doc, tf) of [(doc ids ascending, tfs)]."""
    off = np.zeros(len(lists) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d, _ in lists])
    cat = lambda xs: np.concatenate([np.asarray(x, np.uint32) for x in xs]) if xs else np.zeros(0, np.uint32)
    return off, cat([d for d, _ in lists]), cat([t for _, t in lists])


# ---- champion edge corpus ----

LENGTHS = [1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 224, 225, 256, 257, 1000, 100_000]
N_EDGE = 120_000
TF_MAX = (1 << 24) - 1


def _edge_terms(rng, N, lengths):
    """(pattern, doc ids, tfs) per posting-list length.  Doc order is scan order: k_champions buffers postings in doc order
    and cuts the buffer back to 128 when it holds more than 224, so positions 224..256 of a list are where cuts fall."""
    out = []
    for L in lengths:
        ends = np.array([0, N - 1])[:min(L, 2)]                  # postings on doc 0 and on doc N - 1
        docs = np.sort(np.r_[ends, 1 + rng.choice(N - 2, size=L - len(ends), replace=False)]).astype(np.uint32)
        out.append(("rising", docs, np.arange(1, L + 1)))        # every posting beats the threshold: a cut every round
        out.append(("falling", docs, np.arange(L, 0, -1)))
        out.append(("equal", docs, np.ones(L, np.int64)))        # b = 0: one tie group, the first 128 doc ids
        if L == 1:
            out.append(("last", np.array([N - 1], np.uint32), np.ones(1, np.int64)))
        if L > CHAMP_L:                                          # a tie group over ranks 100 .. 159 (rank 128 inside)
            tf = np.ones(L, np.int64)
            pos = rng.permutation(L)
            tf[pos[:100]] = 9
            tf[pos[100:160]] = 5
            out.append(("tie128", docs, tf))
        if L > 256:                                              # buffer positions 200 .. 279 tie, the first cut inside
            tf = np.ones(L, np.int64)
            tf[0:200:2] = 9
            tf[200:280] = 5
            out.append(("tie224", docs, tf))
        if L >= 5:                                               # the largest tf a posting can hold
            tf = rng.integers(1, 1000, size=L)
            tf[rng.choice(L, size=max(1, L // 6), replace=False)] = TF_MAX
            out.append(("tfmax", docs, tf))
    out.append(("tfmax_all", np.sort(rng.choice(N, size=300, replace=False)).astype(np.uint32), np.full(300, TF_MAX)))
    return out


def _near_tie_term(orc, rng, N, doc_len, k1, b, n_pairs=40):
    """A term whose list order depends on the last bits of s1: pairs of postings (tf, fieldnorm) whose exact scores
    (tf·s0)/(tf + s1[fn]) rank one way and rank the other way with s1 rounded to f32.  Its champion list is its whole
    list (df = 2·n_pairs <= 128), so a kernel that scores with the f32 table lists it in another order."""
    fn = fieldnorms(orc, doc_len)
    avgdl = float(int(np.asarray(doc_len, np.uint64).sum())) / N
    s0, s1 = cache(orc, N, [2 * n_pairs], k1, b, avgdl)
    s1f = s1.astype(np.float32).astype(np.float64)
    present = np.unique(fn)
    tf, f = [a.ravel() for a in np.meshgrid(np.arange(1, 4097), present)]
    sd = (tf * s0[0]) / (tf + s1[f])
    sf = (tf * s0[0]) / (tf + s1f[f])
    order = np.argsort(-sd, kind="stable")
    a, c = order[:-1], order[1:]
    inv = np.flatnonzero((sd[a] > sd[c]) & (sf[a] < sf[c]))
    used, pairs = set(), []
    for i in rng.permutation(inv):
        if a[i] in used or c[i] in used:
            continue
        used.update((a[i], c[i]))
        pairs.append((a[i], c[i]))
        if len(pairs) == n_pairs:
            break
    assert len(pairs) == n_pairs, f"only {len(pairs)} score pairs that f32 s1 reorders"
    docs_of = {int(x): list(rng.permutation(np.flatnonzero(fn == x))) for x in present}
    post = {}
    for p, q in pairs:
        for j in (p, q):
            d = docs_of[int(f[j])].pop()                         # a document with that norm, not used yet
            post[int(d)] = int(tf[j])
    docs = np.array(sorted(post), np.uint32)
    return docs, np.array([post[int(d)] for d in docs], np.int64)


@pytest.fixture(scope="module")
def edge_corpus(m, orc):
    """Edge terms, then fillers, then the edge terms again at ordinals >= sm_count x 64: the grid of k_champions is at
    most sm_count x 16 blocks of 4 warps, so that second copy is scanned by warps whose buffers already held a list."""
    rng = np.random.default_rng(0xC4A)
    N = N_EDGE
    doc_len = rng.integers(1, 3000, size=N).astype(np.uint32)   # lengths over ~150 distinct fieldnorms (b > 0)
    first = _edge_terms(rng, N, [L for L in LENGTHS if L <= 1000])
    second = _edge_terms(rng, N, LENGTHS)
    warps = sm_count() * 64
    fill = []
    for _ in range(warps - len(first) - 1):
        d = np.sort(rng.choice(N, size=int(rng.integers(1, 5)), replace=False)).astype(np.uint32)
        fill.append(("fill", d, rng.integers(1, 4, size=len(d))))
    near = ("near_tie", *_near_tie_term(orc, rng, N, doc_len, 1.2, 0.75))
    terms = first + [near] + fill + second
    assert len(terms) > warps and len(first) + 1 + len(fill) == warps
    off, doc, tf = _csr([(d, t) for _, d, t in terms])
    assert 5e5 < len(doc) < 1.5e6
    return dict(N=N, doc_len=doc_len, off=off, doc=doc, tf=tf, names=[n for n, _, _ in terms], warps=warps)


def _champ_docs(r, t):
    lo, hi = int(r.champ_off[t]), int(r.champ_off[t + 1])
    return r.champ.reshape(-1, 2)[lo:hi, 0]


@pytest.mark.parametrize("k1,b", [(1.2, 0.0), (1.2, 0.75)], ids=["b=0", "b=0.75"])
def test_champion_edge_corpus(m, orc, edge_corpus, k1, b):
    """List lengths around the buffer (224 / 256) and the list length (128), rising and falling scores along doc order,
    one tie group per list (b = 0), tie groups over rank 128 and over the first cut, tf = 2^24 - 1, postings on the first
    and last document, more terms than warps — and, with b > 0, a list whose order only the f64 s1 table gets right."""
    e = edge_corpus
    N, off = e["N"], e["off"]
    assert off[-1] > 0 and len(e["names"]) > sm_count() * 64
    ix = m.Index(N, e["doc_len"], len(off) - 1, off, e["doc"], e["tf"], k1=k1, b=b)
    r = restate(orc, N, off, e["doc"], e["tf"], k1, b, doc_len=e["doc_len"])
    # the restatement states what each pattern's list must be
    o = off.astype(np.int64)
    for t, name in enumerate(e["names"]):
        docs = e["doc"][o[t]:o[t + 1]]
        want = {"rising": docs[::-1], "falling": docs, "equal": docs}.get(name)
        if b == 0 and want is not None:   # b = 0: the score is a function of tf alone
            assert np.array_equal(_champ_docs(r, t), want[:CHAMP_L]), (t, name)
    near = e["names"].index("near_tie")
    s1f = r.s1f.astype(np.float64)
    d = e["doc"][o[near]:o[near + 1]].astype(np.int64)
    tf = e["tf"][o[near]:o[near + 1]].astype(np.float64)
    fn = r.fieldnorm[d]
    sf = (tf * r.s0d[near]) / (tf + s1f[fn])
    f32_order = d[np.lexsort((d, -sf))]
    assert np.array_equal(np.sort(_champ_docs(r, near)), np.sort(d))
    assert (b == 0) == np.array_equal(_champ_docs(r, near), f32_order), "near-tie list not sensitive to s1's rounding"
    _check(ix, r, f"edge corpus k1={k1} b={b}")
    ix.close()


CREATE = dict(varlen=(21, 20000, 3000, 1, 300, 0.0, 1.2, 0.75), b0=(261, 20000, 2000, 1, 200, 0.8, 1.2, 0.0),
              k1_2_b1=(271, 20000, 2500, 1, 250, 0.5, 2.0, 1.0))


@pytest.mark.parametrize("shape", list(CREATE))
def test_create(m, orc, shape):
    seed, n, vocab, lmin, lmax, zipf, k1, b = CREATE[shape]
    c = m.synth_corpus(seed, n, vocab, lmin, lmax, zipf)
    ix = m.Index(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, k1=k1, b=b)
    r = restate(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, k1, b, doc_len=c.doc_len)
    assert np.count_nonzero(r.df > 256) > 50      # lists the buffer is cut on
    _check(ix, r, f"create {shape}")
    ix.close()


def test_stored_blocks_both_norm_forms(m, orc):
    """bm25x_index_create_from_blocks with exact lengths and with stored norms + Σ length: every array byte-equal to the
    plain build's, derived arrays included, and to the restatement."""
    c = m.synth_corpus(43, 20000, 300, 4, 200, 0.7)
    eb = orc.EncodedBlocks(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf))
    fn = fieldnorms(orc, c.doc_len)
    total = int(c.doc_len.astype(np.uint64).sum())
    plain = m.Index.from_corpus(c)
    r = restate(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, 1.2, 0.75, doc_len=c.doc_len)
    want = _check(plain, r, "plain")
    for name, kw in (("doc_len", dict(doc_len=c.doc_len)), ("fieldnorm", dict(doc_fieldnorm=fn, sum_doc_len=total))):
        ix = m.Index.from_blocks(c.n_docs, c.n_terms, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf,
                                 eb.doc_off, eb.tf_off, eb.bytes[:eb.n_bytes], **kw)
        got = _check(ix, r, f"blocks {name}")
        for key in want:
            assert want[key].tobytes() == got[key].tobytes(), f"blocks {name}: {key} differs from the plain build"
        ix.close()
    plain.close()


def _same_shape(rng, c):
    """Another corpus with the same N and the same df per term: other doc ids, other tfs, other lengths."""
    df = np.diff(c.post_off.astype(np.int64))
    lists = [(np.sort(rng.choice(c.n_docs, size=int(n), replace=False)), rng.integers(1, 9, size=int(n))) for n in df]
    off, doc, tf = _csr(lists)
    doc_len = (np.bincount(doc, weights=tf, minlength=c.n_docs) + rng.integers(0, 40, size=c.n_docs)).astype(np.uint32)
    return off, doc, tf, np.maximum(doc_len, 1)


def test_replica_refinalized(m, orc):
    """A replica on the source's device: after finalize_replica its derived arrays are the source's.  Then its arrays are
    refilled from another corpus of the same shape and it is finalized again: every array must be that corpus's,
    champion lists included, and its seeded searches those of an index built from it."""
    rt = cudart()
    c = m.synth_corpus(95, 30000, 5000, 8, 48, 1.0)   # lists from a few postings to most documents
    src = m.Index.from_corpus(c)
    lay = src.layout()
    rep = m.Index.alloc_replica(lay, 0)
    assert rep.derived().n_champ == 0 and not rep.derived().champ  # not finalized: no champion lists yet

    def fill(from_lay):
        rl = rep.layout()
        for i in range(len(rl.dev_ptr)):
            assert rl.bytes[i] == from_lay.bytes[i]
            assert rt.cudaMemcpy(rl.dev_ptr[i], from_lay.dev_ptr[i], from_lay.bytes[i], D2D) == 0
        rep.finalize_replica()

    fill(lay)
    r = restate(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, 1.2, 0.75, doc_len=c.doc_len)
    want = _check(src, r, "replica source")
    got = _check(rep, r, "replica")
    for key in ("pdoc", "champ", "champ_off"):
        assert want[key].tobytes() == got[key].tobytes(), key
    assert rep.derived().s1f_min == src.derived().s1f_min

    off2, doc2, tf2, len2 = _same_shape(np.random.default_rng(96), c)
    ix2 = m.Index(c.n_docs, len2, c.n_terms, off2, doc2, tf2)
    fill(ix2.layout())
    r2 = restate(orc, c.n_docs, off2, doc2, tf2, 1.2, 0.75, doc_len=len2)
    # the replica keeps the scalars it was allocated with (sum of lengths, avgdl); its arrays are the new corpus's
    _check(rep, r2, "replica refilled and finalized again", skip=("sum_doc_len", "avgdl"))
    # a third fill whose lists are one posting longer where that keeps the padded lengths and the block counts: the
    # champion lists change length, so finalize allocates them again
    df2 = np.diff(off2.astype(np.int64))
    grow = (df2 % 4 != 0) & (df2 % 128 != 0) & (df2 < CHAMP_L)
    assert grow.sum() > 100
    rng = np.random.default_rng(98)
    lists = []
    for t, n in enumerate(df2 + grow):
        lists.append((np.sort(rng.choice(c.n_docs, size=int(n), replace=False)), rng.integers(1, 9, size=int(n))))
    off3, doc3, tf3 = _csr(lists)
    ix3 = m.Index(c.n_docs, len2, c.n_terms, off3, doc3, tf3)
    fill(ix3.layout())
    r3 = restate(orc, c.n_docs, off3, doc3, tf3, 1.2, 0.75, doc_len=len2)
    assert r3.n_champ != r2.n_champ
    _check(rep, r3, "replica with longer lists", skip=("sum_doc_len", "avgdl", "n_postings"))
    ix3.close()
    # and back to the second corpus: its searches, seeded, on the replica and on an index built from it
    fill(ix2.layout())
    _check(rep, r2, "replica refilled a third time", skip=("sum_doc_len", "avgdl"))
    q_off, q_terms = m.synth_queries(97, 200, c.n_terms, 2, 4, off2, 0.0)
    for idx in (rep, ix2):
        for name, v in dict(seed=1, seed_dense_div=0, seed_prune_min=0xFFFFFFFF).items():
            idx.set_option(name, v)
    for k in (1, 10, 100):
        a, b = ix2.search_batch(q_off, q_terms, k), rep.search_batch(q_off, q_terms, k)
        for key in ("doc", "score64", "n"):
            assert np.array_equal(a[key], b[key]), (key, k)
    rep.close()
    ix2.close()
    src.close()


def _growing_csr(g, T, sealed_df):
    """The growing documents inverted, as search.rs:83-135 sees them: no posting from a deleted document, from a token the
    sealed segment does not know, or from a term with no sealed posting."""
    n = len(g.elem_off) - 1
    owner = np.repeat(np.arange(n), np.diff(g.elem_off.astype(np.int64)))
    term = g.elem_term.astype(np.int64)
    keep = (g.deleted[owner] == 0) & (term < T)
    keep[keep] = sealed_df[term[keep]] > 0
    t, d, tf = term[keep], owner[keep], g.elem_tf[keep]
    order = np.lexsort((d, t))
    off = np.zeros(T + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(t, minlength=T))
    return off, d[order].astype(np.uint32), tf[order].astype(np.uint32)


def test_growing_handle(m, orc):
    """bm25x_growing_create scores with the sealed segment's N, df and avgdl: its arrays against the restatement of its
    inverted documents with those statistics — norms from exact lengths and from stored norms, synthetic ctids of the
    growing ordinal and explicit ones."""
    sealed = m.synth_corpus(61, 20000, 3000, 8, 80, 0.8)
    fresh = orc.Corpus.synth(62, 2500, 3200, 1, 300, zipf_s=0.8)
    G = fresh.n_docs
    deleted = (np.arange(G) % 5 == 2).astype(np.uint8)
    g = orc.GrowingDocs.from_corpus(fresh, deleted)
    g.elem_term = np.where(g.elem_term >= sealed.n_terms, m.TERM_MISSING, g.elem_term).astype(np.uint32)
    assert np.count_nonzero(g.elem_term == m.TERM_MISSING) > 100
    ix = m.Index.from_corpus(sealed)
    sdf = ix.df()
    stat = (sealed.n_docs, sdf, float(int(sealed.doc_len.astype(np.uint64).sum())) / sealed.n_docs)
    off, doc, tf = _growing_csr(g, sealed.n_terms, sdf)
    assert np.count_nonzero(np.diff(off.astype(np.int64)) > 256) > 5
    fn = fieldnorms(orc, g.doc_len)
    ctid = np.random.default_rng(62).integers(0, 65535, size=(G, 3)).astype(np.uint16)
    for name, kw, rkw, skip in (
            ("doc_len", dict(doc_len=g.doc_len), dict(doc_len=g.doc_len), ()),
            # stored norms carry no length total: the growing handle scores with the sealed avgdl and keeps none
            ("fieldnorm+ctid", dict(doc_fieldnorm=fn, payload=ctid), dict(fieldnorm=fn, sum_len=0, payload=ctid),
             ("sum_doc_len",))):
        gix = ix.growing(g.elem_off, g.elem_term, g.elem_tf, deleted=deleted, **kw)
        r = restate(orc, G, off, doc, tf, 1.2, 0.75, stat=stat, **rkw)
        got = _check(gix, r, f"growing {name}", skip)
        live = got["post"].reshape(-1, 2)[:, 0]
        live = live[live != 0xFFFFFFFF]
        assert len(live) == len(doc) and not np.any(deleted[live]), "a deleted document holds postings"
        gix.close()
    ix.close()


def _local_csr(off, doc, tf, lo, hi):
    o = off.astype(np.int64)
    term = np.repeat(np.arange(len(o) - 1), np.diff(o))
    keep = (doc >= lo) & (doc < hi)
    loff = np.zeros(len(o), np.uint64)
    loff[1:] = np.cumsum(np.bincount(term[keep], minlength=len(o) - 1))
    return loff, (doc[keep] - lo).astype(np.uint32), tf[keep]


def _check_shards(m, orc, c, sx, ix, k1, b, what):
    """Every shard against the restatement of its local CSR with the whole segment's statistics; its score tables
    byte-equal to the unsharded index's; its champion lists the whole ranking of each term restricted to its documents."""
    N, T = int(c["n_docs"]), int(c["n_terms"])
    off, doc, tf = c["post_off"], np.asarray(c["post_doc"]), np.asarray(c["post_tf"])
    df = np.diff(off.astype(np.int64))
    stat = (N, df, float(int(np.asarray(c["doc_len"], np.uint64).sum())) / N)
    whole = read_back(ix.layout(), ix.derived())
    rw = restate(orc, N, off, doc, tf, k1, b, doc_len=c["doc_len"])
    bounds = sx.doc_bounds()
    for s in range(len(bounds) - 1):
        lo, hi = int(bounds[s]), int(bounds[s + 1])
        lay, der = sx.shard_arrays(s)
        got = read_back(lay, der)
        loff, ldoc, ltf = _local_csr(off, doc, tf, lo, hi)
        r = restate(orc, hi - lo, loff, ldoc, ltf, k1, b, doc_len=c["doc_len"][lo:hi], stat=stat, doc_base=lo)
        assert_matches(got, lay, der, r, f"{what} shard {s} [{lo}, {hi})")
        for key in ("s0d", "s0f", "s1d", "s1f"):
            assert got[key].tobytes() == whole[key].tobytes(), f"{what} shard {s}: {key} differs from the whole index's"
        inside = (doc >= lo) & (doc < hi)
        sub = np.flatnonzero(inside)
        champ, champ_off = champion_lists(rw.term[sub], doc[sub].astype(np.int64) - lo, (tf[sub].astype(np.int64) << 8) |
                                          rw.fieldnorm[doc[sub]], rw.score[sub], np.bincount(rw.term[sub], minlength=T))
        assert np.array_equal(got["champ_off"], champ_off), f"{what} shard {s}: champion offsets"
        assert np.array_equal(got["champ"], champ.reshape(-1)), f"{what} shard {s}: not the whole ranking restricted"


@pytest.mark.parametrize("S", [1, 3, 16])
def test_shards_default_bounds(m, orc, S):
    c = m.synth_corpus(71, 30000, 2000, 4, 120, 0.8)
    cd = dict(n_docs=c.n_docs, doc_len=c.doc_len, n_terms=c.n_terms, post_off=c.post_off, post_doc=c.post_doc,
              post_tf=c.post_tf)
    ix = m.Index(**cd)
    sx = m.ShardedIndex(**cd, n_shards=S)
    _check_shards(m, orc, cd, sx, ix, 1.2, 0.75, f"S={S}")
    with pytest.raises(m.Bm25xError) as e:
        sx.shard_arrays(S)
    assert e.value.code == 1 and f"shard {S} of {S}" in str(e.value)
    sx.close()
    ix.close()


def test_shards_adversarial_bounds(m, orc):
    """The bounds of test_gpu_sharded.py::test_adversarial_bounds: a one-document shard, a shard with no postings."""
    from test_gpu_sharded import ADVERSARIAL_BOUNDS, _adversarial_corpus
    c, _ = _adversarial_corpus()
    ix = m.Index(**c)
    sx = m.ShardedIndex(**c, n_shards=len(ADVERSARIAL_BOUNDS) - 1, doc_bounds=ADVERSARIAL_BOUNDS)
    _check_shards(m, orc, c, sx, ix, 1.2, 0.75, "adversarial")
    sx.close()
    ix.close()
