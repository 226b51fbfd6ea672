"""CPU restatement of an index handle's device arrays, for tests that read them back and compare bit for bit.

From a term-major CSR corpus, k1 and b it gives the 13 arrays every handle holds (bm25x_index_layout: postings with the
fieldnorm folded in, offsets, block descriptors, score tables, score bounds, norms, payloads) and the ones a handle derives
on its own device and never replicates (bm25x_index_derived: the doc-id copy `pdoc`, the champion lists, s1f_min).
A growing segment scores with its sealed segment's statistics and a document shard with its whole segment's: `stat`
overrides N, df and avgdl as BuildMeta.stat_* does, and `doc_base` shifts the synthetic payload of a shard's local ids.
Cache (s0 per term, s1 per fieldnorm) comes from the oracle's C code; every other value is numpy."""
import ctypes as C
from types import SimpleNamespace

import numpy as np

from util_cuda import download

# the 13 arrays of bm25x_index_layout, in dev_ptr order
LAYOUT = [("post", np.uint32), ("post_off", np.uint64), ("df", np.uint32), ("blk_off", np.uint64), ("blk", np.uint32),
          ("s0f", np.float32), ("s0d", np.float64), ("s1d", np.float64), ("s1f", np.float32), ("fieldnorm", np.uint8),
          ("payload", np.uint16), ("ubd", np.float64), ("blk_ub", np.float32)]
DERIVED = [("pdoc", np.uint32), ("champ", np.uint32), ("champ_off", np.uint64)]
INFLATE = np.float64(1.0 + 2.0 ** -40)
CHAMP_L = 128
ALIGN, SLACK, BLOCK = 4, 4, 128
CTID_PER_PAGE = 291  # synthetic payload: (block hi, block lo, offset) of a 291-tuple page


def f32_up(x):
    """Smallest f32 >= each f64 of x."""
    f = x.astype(np.float32)
    low = f.astype(np.float64) < x
    f[low] = np.nextafter(f[low], np.float32(np.inf))
    return f


def fieldnorms(orc, doc_len):
    """Quantised norm of each length (bm25.rs:278-283): the last table entry <= the length.  Checked against the oracle's
    C function on a sample."""
    L = orc.lib()
    table = np.array([L.orc_fieldnorm_to_length(f) for f in range(256)], dtype=np.int64)
    doc_len = np.asarray(doc_len, dtype=np.int64)
    fn = (np.searchsorted(table, doc_len, side="right") - 1).astype(np.uint8)
    for d in np.random.default_rng(1).choice(len(doc_len), size=min(len(doc_len), 200), replace=False):
        assert fn[d] == L.orc_length_to_fieldnorm(int(doc_len[d])), (d, doc_len[d])
    return fn


def ctid(ids):
    """Synthetic payload of the given (global) doc ids, [len(ids), 3] u16."""
    g = np.asarray(ids, dtype=np.int64)
    blkno = g // CTID_PER_PAGE
    return np.stack([blkno >> 16, blkno & 0xFFFF, g % CTID_PER_PAGE + 1], axis=1).astype(np.uint16)


def synthetic_payload(n_docs, doc_base=0):
    return ctid(np.arange(n_docs, dtype=np.int64) + doc_base).reshape(-1)


def cache(orc, n_docs, df, k1, b, avgdl):
    """(s0[n_terms], s1[256]) of the oracle's Cache::new (bm25.rs:340-354) for every term."""
    L = orc.lib()
    s0 = np.zeros(len(df))
    s1 = (C.c_double * 256)()
    s0_t = C.c_double()
    for t in range(len(df)):
        L.orc_cache_new(int(n_docs), int(df[t]), float(k1), float(b), float(avgdl), C.byref(s0_t), s1)
        s0[t] = s0_t.value
    return s0, np.array(s1[:])


def champion_lists(term, doc, w, score, df):
    """Per term its best min(df, 128) postings, f64 score descending then doc id ascending: (champ [n, 2] u32 of
    (doc, w), champ_off [T + 1])."""
    off = np.concatenate([[0], np.cumsum(df)]).astype(np.int64)
    order = np.lexsort((doc, -score, term))  # term ascending, then score descending, then doc ascending
    rank = np.arange(len(term)) - off[term]  # order keeps every term's postings where they were: term[order] == term
    keep = order[rank < CHAMP_L]
    champ = np.stack([doc[keep], w[keep]], axis=1).astype(np.uint32)
    champ_off = np.concatenate([[0], np.cumsum(np.minimum(df, CHAMP_L))]).astype(np.uint64)
    return champ, champ_off


def restate(orc, n_docs, post_off, post_doc, post_tf, k1, b, *, doc_len=None, fieldnorm=None, sum_len=None, stat=None,
            doc_base=0, payload=None):
    """Every array of a handle built from this CSR.  Norms from exact lengths (`doc_len`) or, as stored pages hold them,
    from `fieldnorm` + `sum_len`.  stat = (n_docs, df[n_terms], avgdl) the handle scores with, or None for its own.
    Returns a namespace: the arrays under their LAYOUT / DERIVED names (flat, in the dtype they are read back in), the
    layout's scalars, s1f_min, and per posting its term and exact score (for the score-bound checks)."""
    N = int(n_docs)
    if doc_len is not None:
        fn = fieldnorms(orc, doc_len)
        sum_len = int(np.asarray(doc_len, dtype=np.uint64).sum())
    else:
        fn = np.asarray(fieldnorm, dtype=np.uint8)
    assert len(fn) == N
    doc = np.asarray(post_doc, dtype=np.int64)
    r = restate_postings(orc, N, post_off, post_doc, post_tf, fn[doc], np.unique(fn), k1, b, sum_len, stat=stat)
    r.fieldnorm = fn
    r.payload = np.asarray(payload, dtype=np.uint16).reshape(-1) if payload is not None else synthetic_payload(N, doc_base)
    return r


def restate_postings(orc, n_docs, post_off, post_doc, post_tf, post_fn, norms_present, k1, b, sum_len, stat=None):
    """The arrays restate() gives that the postings alone determine (all but fieldnorm and payload), at a cost in the
    number of postings, whatever n_docs: post_fn is the fieldnorm of each posting's document, norms_present the distinct
    fieldnorms of all documents (for s1f_min)."""
    N = int(n_docs)
    off = np.asarray(post_off, dtype=np.int64)
    doc = np.asarray(post_doc, dtype=np.int64)
    tf = np.asarray(post_tf, dtype=np.int64)
    pfn = np.asarray(post_fn, dtype=np.uint8)
    T, P = len(off) - 1, int(off[-1])
    df = np.diff(off)
    avgdl = float(stat[2]) if stat is not None else float(sum_len) / float(N)
    s0, s1 = cache(orc, stat[0] if stat is not None else N, stat[1] if stat is not None else df, k1, b, avgdl)
    r = SimpleNamespace(n_docs=N, n_terms=T, n_postings=P, sum_doc_len=sum_len, avgdl=avgdl, k1=float(k1), b=float(b))

    # postings: (doc, tf << 8 | fieldnorm) in CSR order, each list padded with {0xFFFFFFFF, 0} to a multiple of 4 slots,
    # then the slack slots (all ones)
    term = np.repeat(np.arange(T), df)
    w = (tf << 8) | pfn.astype(np.int64)
    pad = (df + ALIGN - 1) // ALIGN * ALIGN
    off_pad = np.concatenate([[0], np.cumsum(pad)]).astype(np.int64)
    pos = off_pad[term] + (np.arange(P) - off[term])
    post = np.zeros((off_pad[-1] + SLACK, 2), dtype=np.uint32)
    post[:, 0] = 0xFFFFFFFF
    post[off_pad[-1]:, 1] = 0xFFFFFFFF
    post[pos, 0] = doc
    post[pos, 1] = w
    r.n_postings_padded = int(off_pad[-1])
    r.post, r.post_off, r.df = post.reshape(-1), off_pad.astype(np.uint64), df.astype(np.uint32)
    r.pdoc = post[:, 0].copy()

    # blocks of 128 postings: offsets, (first doc, last doc)
    nb = (df + BLOCK - 1) // BLOCK
    blk_off = np.concatenate([[0], np.cumsum(nb)]).astype(np.int64)
    r.n_blocks = int(blk_off[-1])
    bterm = np.repeat(np.arange(T), nb)
    start = off[bterm] + BLOCK * (np.arange(r.n_blocks) - blk_off[bterm])
    end = np.minimum(start + BLOCK, off[bterm + 1])
    r.blk_off = blk_off.astype(np.uint64)
    r.blk = np.stack([doc[start], doc[end - 1]], axis=1).astype(np.uint32).reshape(-1)

    r.s0d, r.s0f, r.s1d, r.s1f = s0, s0.astype(np.float32), s1, s1.astype(np.float32)

    # every posting's exact score, Cache::evaluate's operation order (checked against the C function on a sample)
    tfd = tf.astype(np.float64)
    score = (tfd * s0[term]) / (tfd + s1[pfn])
    s1c = (C.c_double * 256)(*s1)
    for p in np.random.default_rng(0).choice(P, size=min(P, 300), replace=False):
        assert score[p] == orc.lib().orc_cache_evaluate(s0[term[p]], s1c, int(pfn[p]), int(tf[p]))
    r.term, r.score, r.blk_start, r.blk_term = term, score, start, bterm
    # score bounds: ubd = (best single-posting score) x (1 + 2^-40), blk_ub = the smallest f32 >= (block max) x (1 + 2^-40)
    tmax = np.zeros(T)
    tmax[df > 0] = np.maximum.reduceat(score, off[:-1][df > 0]) if P else 0.0
    r.ubd = tmax * INFLATE
    r.block_max = np.maximum.reduceat(score, start) if r.n_blocks else np.zeros(0)
    r.blk_ub = f32_up(r.block_max * INFLATE)

    r.champ, r.champ_off = champion_lists(term, doc, w, score, df)
    r.champ = r.champ.reshape(-1)
    r.n_champ = int(r.champ_off[-1])
    r.s1f_min = np.float32(r.s1f[np.asarray(norms_present, dtype=np.int64)].min())
    return r


def read_back(lay, der):
    """A handle's arrays as the device holds them: the 13 of `lay` (IndexLayout) and those of `der` (IndexDerived)."""
    got = {name: download(lay.dev_ptr[i], lay.bytes[i], dt) for i, (name, dt) in enumerate(LAYOUT)}
    for name, dt in DERIVED:
        n = int(getattr(der, name + "_bytes"))
        got[name] = download(getattr(der, name), n, dt) if n else np.zeros(0, dt)
    return got


SCALARS = ("n_docs", "n_terms", "n_postings", "n_postings_padded", "n_blocks", "sum_doc_len", "k1", "b", "avgdl")


def assert_matches(got, lay, der, r, what, skip=()):
    """Every array and scalar of a handle against the restatement, bit for bit.  An array the restatement leaves empty
    (no blocks) is one placeholder slot on the device, whose content is not specified."""
    for name in SCALARS:
        if name not in skip:
            assert getattr(lay, name) == getattr(r, name), f"{what}: layout.{name} {getattr(lay, name)} != {getattr(r, name)}"
    assert der.n_champ == r.n_champ, f"{what}: n_champ {der.n_champ} != {r.n_champ}"
    assert der.s1f_min == r.s1f_min, f"{what}: s1f_min {der.s1f_min} != {r.s1f_min}"
    for name, _ in LAYOUT + DERIVED:
        if name in skip:
            continue
        want, have = getattr(r, name), got[name]
        if want.size == 0 and have.nbytes <= 8:
            continue
        assert have.shape == want.shape, f"{what}: {name} holds {have.shape} entries, restatement {want.shape}"
        if not np.array_equal(have, want):
            bad = np.flatnonzero(have != want)
            raise AssertionError(f"{what}: {name} differs at {len(bad)} entries, first {bad[:4].tolist()}: "
                                 f"device {have[bad[:4]].tolist()} restatement {want[bad[:4]].tolist()}")
