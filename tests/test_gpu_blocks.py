"""GPU: ingest of the reference's stored posting blocks (SURVEY §8 f1, bm25x_index_create_from_blocks).

The oracle's codec restatement (oracle/bm25_codec.c, pinned in tests/test_codec.py) encodes a corpus the way flush.rs
does; the product decodes the blocks on the GPU.  Bar: the decoded index is byte-identical to the one built from the
plain postings (all 13 device arrays), and searches on it are bit-exact against the oracle."""
import numpy as np
import pytest

from util_corpora import BLOCK_CONFIGS
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import compare, oracle_index

pytestmark = pytest.mark.gpu


def _device_arrays(ix):
    import torch
    lay = ix.layout()
    out = []
    for i in range(len(lay.bytes)):
        n = int(lay.bytes[i])
        if n == 0:
            out.append(np.zeros(0, dtype=np.uint8))
            continue
        view = type("DevArray", (), {"__cuda_array_interface__": {
            "shape": (n,), "typestr": "|u1", "data": (int(lay.dev_ptr[i]), False), "version": 3}})()
        out.append(torch.as_tensor(view, device="cuda:0").cpu().numpy().copy())
    return out


def _from_blocks(m, orc, c, **kw):
    eb = orc.EncodedBlocks(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf))
    args = dict(doc_len=c.doc_len)
    args.update(kw)
    return eb, m.Index.from_blocks(c.n_docs, c.n_terms, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf,
                                   eb.doc_off, eb.tf_off, eb.bytes[:eb.n_bytes], **args)


@pytest.mark.parametrize("cfg", BLOCK_CONFIGS, ids=[c["name"] for c in BLOCK_CONFIGS])
def test_blocks_index_identical_and_search_exact(m, orc, cfg):
    c = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    plain = m.Index.from_corpus(c)
    eb, ix = _from_blocks(m, orc, c)
    assert ix.info().n_postings == plain.info().n_postings and ix.info().n_blocks == eb.n_blocks
    for i, (a, b) in enumerate(zip(_device_arrays(plain), _device_arrays(ix))):
        assert np.array_equal(a, b), f"{cfg['name']}: device array {i} differs between CSR build and block ingest"
    q_off, q_terms = m.synth_queries(cfg["seed"] + 1000, 40, cfg["vocab"], 1, 8, c.post_off, cfg["zipf"])
    oix = oracle_index(orc, c)
    for k in (1, 10, 100):
        compare(ix.search_batch(q_off, q_terms, k), oix, q_off, q_terms, k, what="blocks-" + cfg["name"])
    plain.close()
    ix.close()


def test_blocks_from_stored_norms(m, orc):
    # the pages hold DocumentTuple.fieldnorm + JumpTuple.sum_of_document_lengths, not exact lengths
    c = m.synth_corpus(41, 4000, 300, 4, 200, 0.7)
    fn = np.array([orc.lib().orc_length_to_fieldnorm(int(x)) for x in c.doc_len], dtype=np.uint8)
    plain = m.Index.from_corpus(c)
    _, ix = _from_blocks(m, orc, c, doc_len=None, doc_fieldnorm=fn, sum_doc_len=int(c.doc_len.astype(np.uint64).sum()))
    for a, b in zip(_device_arrays(plain), _device_arrays(ix)):
        assert np.array_equal(a, b)
    plain.close()
    ix.close()


def test_blocks_wide_deltas_and_tf_limits(m, orc):
    # 26-bit deltas in a full block, 3-byte tf in a short one, tf = 2^24-1 accepted, 2^24 refused.
    # (bit width 32 — raw ids, bitpacking_u32_ordered.rs:119-121 — needs > 2^31 documents: decoded on the GPU by
    # tests/test_gpu_zy_high_doc_ids.py::test_stored_blocks_above_2_31, with a byte-width-4 tail above 2^31.)
    N = 40_000_000
    rng = np.random.default_rng(5)
    docs = np.sort(rng.choice(N, 128 + 77, replace=False)).astype(np.uint32)
    docs[1] = docs[0] + 1
    tfs = rng.integers(1, 1 << 20, len(docs)).astype(np.uint32)
    tfs[3] = (1 << 24) - 1
    tfs[130] = (1 << 24) - 1

    def build(tfs):
        md0, pd0 = orc.compress_document_ids(int(docs[0]), docs[:128])
        mt0, pt0 = orc.compress_term_frequencies(tfs[:128])
        md1, pd1 = orc.compress_document_ids(int(docs[128]), docs[128:])
        mt1, pt1 = orc.compress_term_frequencies(tfs[128:])
        assert md0 >> 7 == 0 and (md0 & 0x7F) >= 20 and mt0 in (24, 25) and md1 >> 7 == 1 and mt1 >> 7 == 1
        data = np.concatenate([pd0, pt0, pd1, pt1])
        offs = np.cumsum([0, len(pd0), len(pt0), len(pd1)])
        return m.Index.from_blocks(N, 1, [0, 2], [docs[0], docs[128]], [128, 77], [md0, md1], [mt0, mt1],
                                   [offs[0], offs[2]], [offs[1], offs[3]], data,
                                   doc_fieldnorm=np.full(N, 20, dtype=np.uint8), sum_doc_len=20 * N)

    ix = build(tfs)
    got_d, got_s = ix.search([0], 1000)
    assert sorted(got_d.tolist()) == docs.tolist()
    # equal norms: the score order is the tf order; the two largest tf are the 2^24-1 ones
    assert set(got_d[:2].tolist()) == {int(docs[3]), int(docs[130])}
    ix.close()
    tfs[50] = 1 << 24
    with pytest.raises(m.Bm25xError, match="2\\^24"):
        build(tfs)


def test_blocks_bytewidth4_tail_is_raw(m, orc):
    """A 77-posting tail block with a gap >= 2^24 is byte-packed with width 4 = raw ids, no delta
    (crates/simd/src/bytepacking_u32_ordered.rs:195,211); routine for rare terms of a 50M-document index."""
    N = 60_000_000
    rng = np.random.default_rng(9)
    head = np.sort(rng.choice(1_000_000, 128, replace=False)).astype(np.uint32)
    first = np.uint32(1_000_007)
    second = np.uint32(int(first) + (1 << 24) + 5)
    rest = np.sort(rng.choice(np.arange(int(second) + 1, N), 75, replace=False)).astype(np.uint32)
    docs = np.concatenate([head, [first, second], rest]).astype(np.uint32)
    tfs = rng.integers(1, 9, len(docs)).astype(np.uint32)
    md0, pd0 = orc.compress_document_ids(int(docs[0]), docs[:128])
    mt0, pt0 = orc.compress_term_frequencies(tfs[:128])
    md1, pd1 = orc.compress_document_ids(int(docs[128]), docs[128:])
    mt1, pt1 = orc.compress_term_frequencies(tfs[128:])
    assert md1 == (0x80 | 4) and len(pd1) == 77 * 4
    assert pd1.view("<u4").tolist() == docs[128:].tolist()          # the payload IS the id list
    data = np.concatenate([pd0, pt0, pd1, pt1])
    offs = np.cumsum([0, len(pd0), len(pt0), len(pd1)])
    ix = m.Index.from_blocks(N, 1, [0, 2], [docs[0], docs[128]], [128, 77], [md0, md1], [mt0, mt1],
                             [offs[0], offs[2]], [offs[1], offs[3]], data,
                             doc_fieldnorm=np.full(N, 20, dtype=np.uint8), sum_doc_len=20 * N)
    got_d, got_s = ix.search([0], 1000)
    assert sorted(got_d.tolist()) == docs.tolist()
    order = np.lexsort((docs, -tfs.astype(np.int64)))               # equal norms: tf desc, then doc id asc
    assert got_d.tolist() == docs[order].tolist()
    ix.close()


def test_blocks_summary_wand_bounds_are_checked(m, orc):
    """SummaryTuple.(wand_fieldnorm, wand_term_frequency) (tuples.rs:900-910, written by flush.rs:101-120): the oracle's
    flush restatement produces them; the ingest accepts the real ones and refuses a pair that is not the block's
    arg-max.  The per-block score bounds of the resulting index equal those of the index built from plain postings
    (device array 12, compared by test_blocks_index_identical_and_search_exact for every config)."""
    c = m.synth_corpus(47, 6000, 60, 4, 120, 0.9)
    oc = orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf)
    wfn, wtf = orc.OracleIndex(oc).block_wand()
    eb, ix = _from_blocks(m, orc, c, blk_wand_fieldnorm=wfn, blk_wand_tf=wtf)
    assert len(wfn) == eb.n_blocks == ix.info().n_blocks
    plain = m.Index.from_corpus(c)
    assert np.array_equal(_device_arrays(plain)[12], _device_arrays(ix)[12])
    ub = _device_arrays(ix)[12].view(np.float32)
    assert len(ub) == eb.n_blocks and np.all(ub > 0)
    plain.close()
    ix.close()
    bad_tf = wtf.copy()
    g = int(np.argmax(wtf))               # a block whose arg-max has tf > 1: halving it lowers the bound
    assert bad_tf[g] > 1
    bad_tf[g] = 1
    with pytest.raises(m.Bm25xError, match="wand"):
        _from_blocks(m, orc, c, blk_wand_fieldnorm=wfn, blk_wand_tf=bad_tf)
    bad_fn = wfn.copy()
    bad_fn[0] = 255 if wfn[0] < 200 else 0   # a very different length norm
    with pytest.raises(m.Bm25xError, match="wand"):
        _from_blocks(m, orc, c, blk_wand_fieldnorm=bad_fn, blk_wand_tf=wtf)


def test_blocks_corruption_is_reported(m, orc):
    c = m.synth_corpus(43, 2000, 20, 8, 40, 0.5)
    eb = orc.EncodedBlocks(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf))

    def build(**over):
        a = dict(term_blk_off=eb.term_blk_off, blk_min_doc=eb.blk_min, blk_n=eb.blk_n, blk_meta_doc=eb.meta_doc,
                 blk_meta_tf=eb.meta_tf, blk_doc_off=eb.doc_off, blk_tf_off=eb.tf_off, data=eb.bytes[:eb.n_bytes])
        a.update(over)
        return m.Index.from_blocks(c.n_docs, c.n_terms, doc_len=c.doc_len, **a)

    build().close()
    t2 = int(np.nonzero(np.diff(eb.term_blk_off.astype(np.int64)) >= 3)[0][0])   # a token with >= 3 blocks
    full = int(eb.term_blk_off[t2])                                              # its first (full, not last) block
    assert eb.blk_n[full] == 128 and eb.blk_n[full + 1] == 128
    # directory errors: caught on the host
    bad_n = eb.blk_n.copy(); bad_n[full] = 100                      # a short block in the middle of a token
    with pytest.raises(m.Bm25xError, match="corrupt block directory"):
        build(blk_n=bad_n)
    bad_meta = eb.meta_doc.copy(); bad_meta[full] = 33               # "bitwidth out of bound"
    with pytest.raises(m.Bm25xError, match="corrupt block metadata"):
        build(blk_meta_doc=bad_meta)
    bad_off = eb.doc_off.copy(); bad_off[full] = eb.n_bytes          # payload past the end
    with pytest.raises(m.Bm25xError, match="corrupt block directory"):
        build(blk_doc_off=bad_off)
    # payload errors: caught by the decoder on the device, never dereferenced
    bad_min = eb.blk_min.copy(); bad_min[full] = c.n_docs            # pushes the doc ids past n_docs
    with pytest.raises(m.Bm25xError, match="corrupt blocks"):
        build(blk_min_doc=bad_min)
    data = eb.bytes[:eb.n_bytes].copy()
    w = int(eb.meta_tf[full]) & 0x7F
    data[int(eb.tf_off[full]):int(eb.tf_off[full]) + 16 * w] = 0    # tf == 0
    with pytest.raises(m.Bm25xError, match="corrupt blocks"):
        build(data=data)
    # the blocks of a token out of order: each block is fine, the chain is not
    b0 = full
    swap = lambda a: np.concatenate([a[:b0], a[b0 + 1:b0 + 2], a[b0:b0 + 1], a[b0 + 2:]])
    with pytest.raises(m.Bm25xError, match="corrupt blocks"):
        build(blk_min_doc=swap(eb.blk_min), blk_meta_doc=swap(eb.meta_doc), blk_meta_tf=swap(eb.meta_tf),
              blk_doc_off=swap(eb.doc_off), blk_tf_off=swap(eb.tf_off))

    # a first delta that wraps: SummaryTuple.min_document_id 0xFFFFFFF0 + 0x20 = document 16 mod 2^32, every later id
    # ascending and < n_docs.  The encoder always writes a first delta of 0, so only a corrupt page holds this; a decoded
    # id below its block's min_document_id contradicts the summary.  Once in a full (bit-packed) block, once in a
    # byte-packed tail.
    N = 1000
    full_docs, tail_docs = 16 + 7 * np.arange(128, dtype=np.uint32), 16 + 5 * np.arange(50, dtype=np.uint32)

    def two_tokens(min_full, min_tail):
        md0, pd0 = orc.compress_document_ids(min_full, full_docs)
        md1, pd1 = orc.compress_document_ids(min_tail, tail_docs)
        mt0, pt0 = orc.compress_term_frequencies(np.ones(128, np.uint32))
        mt1, pt1 = orc.compress_term_frequencies(np.ones(50, np.uint32))
        assert md0 >> 7 == 0 and md0 < 32 and md1 >> 7 == 1 and (md1 & 0x7F) < 4       # delta-coded, both
        data = np.concatenate([pd0, pt0, pd1, pt1])
        offs = np.cumsum([0, len(pd0), len(pt0), len(pd1)])
        return m.Index.from_blocks(N, 2, [0, 1, 2], [min_full, min_tail], [128, 50], [md0, md1], [mt0, mt1],
                                   [offs[0], offs[2]], [offs[1], offs[3]], data,
                                   doc_fieldnorm=np.full(N, 20, dtype=np.uint8), sum_doc_len=20 * N)

    ix = two_tokens(16, 16)                                            # the honest encoding: first delta 0
    assert ix.search([0], 200)[0].tolist() == sorted(full_docs.tolist())
    assert ix.search([1], 200)[0].tolist() == sorted(tail_docs.tolist())
    ix.close()
    wrap = 0xFFFFFFF0
    for mins in ((wrap, 16), (16, wrap)):
        with pytest.raises(m.Bm25xError, match="corrupt blocks"):
            two_tokens(*mins)
