"""numpy restatement of the summaries flush writes beside the block payloads (crates/bm25/src/flush.rs:78-135), and the
expected output of bm25x_index_export_blocks for a term-major CSR corpus.

- Blocks: per term, runs of 128 postings in doc order, the last shorter (flush.rs:78-90).  SummaryTuple: min / max =
  the block's first and last doc id, n its postings, (wand_fieldnorm, wand_term_frequency) = Wand over the block in doc
  order (bm25.rs:297-318): start (tf 0.0, fieldnorm 255, tf 0), a posting replaces it only when its tf() is strictly
  greater, so the first posting of the largest tf() wins.  tf() = (tf·(k1+1)) / (tf + k1·(1−b+b·len(fn)/avgdl))
  (bm25.rs:291-295), in that operation order (numpy never fuses).
- Tokens: df, and Wand::extend over the token's blocks in order (flush.rs:111-112, bm25.rs:319-325): the earliest block
  of the largest tf() wins; a token without postings keeps (255, 0).
The payload bytes and the block directory come from the oracle's codec (oracle.EncodedBlocks).  The oracle's own flush
restatement (orc_index_build) computes every block and token summary too; oracle_summaries() reads them, and
tests/test_export.py pins this restatement against them, ties included."""
import ctypes as C
from types import SimpleNamespace

import numpy as np

BLOCK = 128


class _OrcIndex(C.Structure):
    """struct orc_index of oracle/bm25_oracle.c (x86-64 layout), read-only: the oracle exports its block pairs
    (orc_index_block_wand) but not the rest of the summaries orc_index_build computes.  oracle_summaries() checks the
    mirror against every public accessor on each use, so a change of the oracle's struct fails loudly."""
    _fields_ = [("n_docs", C.c_uint32), ("n_terms", C.c_uint32), ("n_post", C.c_uint64), ("sum_len", C.c_uint64),
                ("k1", C.c_double), ("b", C.c_double), ("avgdl", C.c_double), ("fieldnorm", C.POINTER(C.c_uint8)),
                ("post_off", C.c_void_p), ("post_doc", C.c_void_p), ("post_tf", C.c_void_p),
                ("df", C.POINTER(C.c_uint32)), ("tok_wand_fn", C.POINTER(C.c_uint8)),
                ("tok_wand_tf", C.POINTER(C.c_uint32)), ("sum_off", C.POINTER(C.c_uint64)), ("summaries", C.c_void_p)]


# orc_summary: {u32 min_doc, u32 max_doc, u8 n, u8 wand_fn, u32 wand_tf, u64 first}
_SUMMARY = np.dtype({"names": ["min_doc", "max_doc", "n", "wand_fn", "wand_tf", "first"],
                     "formats": [np.uint32, np.uint32, np.uint8, np.uint8, np.uint32, np.uint64],
                     "offsets": [0, 4, 8, 9, 12, 16], "itemsize": 24})


def oracle_summaries(orc, oix):
    """The SummaryTuple of every block (min_doc, max_doc, n, wand_fn, wand_tf) and the TokenTuple fields of every token
    (df, tok_wand_fn, tok_wand_tf) that the oracle's orc_index_build computed for OracleIndex `oix`, plus blk_off
    (first block of each token).  Copies: valid after oix is freed."""
    L = orc.lib()
    h = oix.h
    ix = C.cast(C.c_void_p(h), C.POINTER(_OrcIndex)).contents
    T = int(ix.n_terms)
    nb = int(L.orc_index_n_blocks(h))
    assert ix.n_docs == L.orc_index_n_docs(h) and ix.avgdl == L.orc_index_avgdl(h), "oracle struct mirror out of date"
    blk_off = np.ctypeslib.as_array(ix.sum_off, shape=(T + 1,)).copy()
    assert int(blk_off[T]) == nb, "oracle struct mirror out of date"
    df = np.ctypeslib.as_array(ix.df, shape=(T,)).copy() if T else np.zeros(0, np.uint32)
    for t in np.unique(np.linspace(0, max(T - 1, 0), min(T, 200)).astype(np.int64)) if T else []:
        assert df[t] == L.orc_index_df(h, int(t)), "oracle struct mirror out of date"
    raw = np.ctypeslib.as_array(C.cast(ix.summaries, C.POINTER(C.c_uint8)), shape=(max(nb, 1) * _SUMMARY.itemsize,))
    sm = raw[:nb * _SUMMARY.itemsize].view(_SUMMARY).copy()
    wfn, wtf = oix.block_wand()
    assert np.array_equal(sm["wand_fn"], wfn) and np.array_equal(sm["wand_tf"], wtf), "oracle struct mirror out of date"
    tok_fn = np.ctypeslib.as_array(ix.tok_wand_fn, shape=(T,)).copy() if T else np.zeros(0, np.uint8)
    tok_tf = np.ctypeslib.as_array(ix.tok_wand_tf, shape=(T,)).copy() if T else np.zeros(0, np.uint32)
    return SimpleNamespace(blk_off=blk_off, min_doc=sm["min_doc"], max_doc=sm["max_doc"], n=sm["n"].astype(np.uint32),
                           wand_fn=sm["wand_fn"], wand_tf=sm["wand_tf"], df=df, tok_wand_fn=tok_fn, tok_wand_tf=tok_tf)


def assert_summaries_match_oracle(orc, got, n_docs, doc_len, post_off, post_doc, post_tf, k1, b, what):
    """An export's block and token summaries against the oracle's flush restatement over the same corpus (exact
    lengths): SummaryTuple min / max / n / wand pair, TokenTuple df / wand pair, term_blk_off."""
    oc = orc.Corpus(n_docs, doc_len, len(post_off) - 1, post_off, post_doc, post_tf, k1=k1, b=b)
    want = oracle_summaries(orc, orc.OracleIndex(oc))
    a, x = got
    for key, have, exp in (("term_blk_off", a["term_blk_off"], want.blk_off), ("blk_min_doc", a["blk_min_doc"], want.min_doc),
                           ("blk_max_doc", x["blk_max_doc"], want.max_doc), ("blk_n", a["blk_n"], want.n),
                           ("blk_wand_fieldnorm", a["blk_wand_fieldnorm"], want.wand_fn),
                           ("blk_wand_tf", a["blk_wand_tf"], want.wand_tf), ("tok_df", x["tok_df"], want.df),
                           ("tok_wand_fieldnorm", x["tok_wand_fieldnorm"], want.tok_wand_fn),
                           ("tok_wand_tf", x["tok_wand_tf"], want.tok_wand_tf)):
        assert np.array_equal(np.asarray(have), exp), f"{what}: {key} differs from the oracle's flush restatement"


def fieldnorm_lengths(orc):
    """len(fn) of every fieldnorm (bm25.rs:274-276), as f64."""
    L = orc.lib()
    return np.array([L.orc_fieldnorm_to_length(f) for f in range(256)], dtype=np.float64)


def tf_values(orc, tf, fn, k1, b, avgdl):
    """tf() of every posting (bm25.rs:291-295)."""
    t = np.asarray(tf, dtype=np.float64)
    dl = fieldnorm_lengths(orc)[np.asarray(fn, dtype=np.int64)]
    return (t * (k1 + 1.0)) / (t + k1 * (1.0 - b + b * dl / avgdl))


def first_argmax(values, starts, n_items):
    """Per segment [starts[i], starts[i + 1]) (the last one ends at n_items; segments non-empty): the index of its first
    largest value."""
    starts = np.asarray(starts, dtype=np.int64)
    if len(starts) == 0:
        return np.zeros(0, np.int64)
    seg = np.repeat(np.arange(len(starts)), np.diff(np.append(starts, n_items)))
    top = np.maximum.reduceat(values, starts)
    cand = np.where(values == top[seg], np.arange(n_items), n_items)
    return np.minimum.reduceat(cand, starts)


def block_summaries(orc, post_off, post_doc, post_tf, post_fn, k1, b, avgdl):
    """Per block (term order) min_doc, max_doc, n, wand_fieldnorm, wand_tf and the pair's tf(); blk_off per term."""
    off = np.asarray(post_off, dtype=np.int64)
    doc, tf, pfn = np.asarray(post_doc), np.asarray(post_tf), np.asarray(post_fn, dtype=np.uint8)
    T, P = len(off) - 1, int(off[-1])
    df = np.diff(off)
    nb = (df + BLOCK - 1) // BLOCK
    blk_off = np.concatenate([[0], np.cumsum(nb)]).astype(np.int64)
    bterm = np.repeat(np.arange(T), nb)
    start = off[bterm] + BLOCK * (np.arange(int(blk_off[-1])) - blk_off[bterm])
    end = np.minimum(start + BLOCK, off[bterm + 1])
    v = tf_values(orc, tf, pfn, k1, b, avgdl)
    win = first_argmax(v, start, P)
    return SimpleNamespace(blk_off=blk_off.astype(np.uint64), min_doc=doc[start].astype(np.uint32),
                           max_doc=doc[end - 1].astype(np.uint32), n=(end - start).astype(np.uint32),
                           wand_fn=pfn[win], wand_tf=tf[win].astype(np.uint32), wand_v=v[win])


def token_wand(blk_off, wand_fn, wand_tf, wand_v):
    """Per token Wand::extend over its blocks: (wand_fieldnorm, wand_tf), (255, 0) without blocks."""
    off = np.asarray(blk_off, dtype=np.int64)
    T = len(off) - 1
    fn, tf = np.full(T, 255, np.uint8), np.zeros(T, np.uint32)
    has = np.diff(off) > 0
    if has.any():
        win = first_argmax(np.asarray(wand_v, dtype=np.float64), off[:-1][has], int(off[-1]))
        fn[has], tf[has] = np.asarray(wand_fn)[win], np.asarray(wand_tf)[win]
    return fn, tf


def expected_export(orc, n_docs, post_off, post_doc, post_tf, k1, b, fieldnorm, sum_len, payload, term_keys=None,
                    post_fn=None):
    """What bm25x_index_export_blocks gives for an index over this CSR with these norms: (args, extra) as
    Index.export_blocks returns them.  post_fn (the fieldnorm of each posting's document) may be given instead of reading
    it from `fieldnorm` (a sparse corpus whose per-document arrays are not exported)."""
    eb = orc.EncodedBlocks(SimpleNamespace(n_terms=len(post_off) - 1, post_off=np.asarray(post_off, np.uint64),
                                       post_doc=np.ascontiguousarray(post_doc, np.uint32),
                                       post_tf=np.ascontiguousarray(post_tf, np.uint32)))
    if post_fn is None:
        post_fn = np.asarray(fieldnorm)[np.asarray(post_doc, dtype=np.int64)]
    s = block_summaries(orc, post_off, post_doc, post_tf, post_fn, k1, b, float(sum_len) / float(n_docs))
    nb = eb.n_blocks
    assert np.array_equal(s.blk_off, eb.term_blk_off) and np.array_equal(s.min_doc, eb.blk_min[:nb])
    assert np.array_equal(s.n, eb.blk_n[:nb])
    tok_fn, tok_tf = token_wand(s.blk_off, s.wand_fn, s.wand_tf, s.wand_v)
    args = dict(n_docs=int(n_docs), n_terms=len(post_off) - 1, term_blk_off=eb.term_blk_off, blk_min_doc=eb.blk_min[:nb],
                blk_n=eb.blk_n[:nb], blk_meta_doc=eb.meta_doc[:nb], blk_meta_tf=eb.meta_tf[:nb],
                blk_doc_off=eb.doc_off[:nb], blk_tf_off=eb.tf_off[:nb], data=eb.bytes[:eb.n_bytes],
                doc_fieldnorm=fieldnorm, sum_doc_len=int(sum_len), k1=float(k1), b=float(b), payload=payload,
                term_keys=term_keys, blk_wand_fieldnorm=s.wand_fn, blk_wand_tf=s.wand_tf)
    extra = dict(blk_max_doc=s.max_doc, tok_df=np.diff(np.asarray(post_off, np.int64)).astype(np.uint32),
                 tok_wand_fieldnorm=tok_fn, tok_wand_tf=tok_tf)
    return args, extra


def assert_export_equal(got, want, what, skip=()):
    """Every output of an export, (args, extra), against the expected one, byte for byte."""
    for g, w in zip(got, want):
        assert set(g) == set(w), what
        for key, e in w.items():
            if key in skip:
                continue
            a = g[key]
            if not isinstance(e, np.ndarray):
                assert a == e, f"{what}: {key} {a} != {e}"
                continue
            a, e = np.asarray(a).reshape(-1), e.reshape(-1)
            assert a.size == e.size, f"{what}: {key} holds {a.size} entries, expected {e.size}"
            if not np.array_equal(a, e):
                bad = np.flatnonzero(a != e)
                raise AssertionError(f"{what}: {key} differs at {len(bad)} entries, first {bad[:4].tolist()}: "
                                     f"export {a[bad[:4]].tolist()} expected {e[bad[:4]].tolist()}")
