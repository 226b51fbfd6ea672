"""CPU: the boundary of the export (bm25x_index_export_blocks): bm25x_export has the layout the C compiler gives the
header, null arguments are refused without touching a device; and the restatement of the summaries flush writes
(util_export, flush.rs:78-135) against the oracle's flush restatement and on small cases derived by hand, ties included."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from util_export import block_summaries, fieldnorm_lengths, oracle_summaries, token_wand
from util_index import fieldnorms
from util_lib import host_library  # noqa: F401  (host_library: the module fixture m)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_export_layout_matches_the_header(m):
    fields = [f for f, _ in m.Export._fields_]
    assert fields == ["doc_fieldnorm", "payload", "sum_doc_len", "term_key", "tok_df", "tok_wand_fieldnorm", "tok_wand_tf",
                      "term_blk_off", "blk_min_doc", "blk_max_doc", "blk_n", "blk_meta_doc", "blk_meta_tf", "blk_doc_off",
                      "blk_tf_off", "blk_wand_fieldnorm", "blk_wand_tf", "bytes", "bytes_cap", "n_bytes"]
    prog = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "bm25x.h")}"',
            "int main(void) {", 'printf("%zu", sizeof(bm25x_export));']
    prog += [f'printf(" %zu", offsetof(bm25x_export, {f}));' for f in fields]
    prog += ["return 0; }"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-std=c11", "-o", exe, src])
        size, *offs = subprocess.check_output([exe], text=True).split()
    assert C.sizeof(m.Export) == int(size)
    assert [getattr(m.Export, f).offset for f in fields] == [int(o) for o in offs]


def test_export_null_arguments_refused(m):
    L = m.load_library()
    e = m.Export()
    e.n_bytes = 77
    for call in (lambda: L.bm25x_index_export_blocks(None, C.byref(e)),
                 lambda: L.bm25x_index_export_blocks(C.c_void_p(8), None)):
        assert call() == 1
        assert L.bm25x_last_error().decode() == "bm25x_index_export_blocks: null argument"
    assert e.n_bytes == 77


def _csr(lists):
    off = np.cumsum([0] + [len(d) for d, _ in lists]).astype(np.uint64)
    doc = np.concatenate([np.asarray(d, np.uint32) for d, _ in lists] + [np.zeros(0, np.uint32)])
    tf = np.concatenate([np.asarray(t, np.uint32) for _, t in lists] + [np.zeros(0, np.uint32)])
    return off, doc, tf


def test_summaries_match_the_oracle(orc):
    """Every block's (min, max, n, wand pair) and every token's (df, wand pair) against the oracle's flush restatement
    (orc_index_build) and its codec's directory, on corpora with blocks of every length and tokens of many blocks; b = 0
    makes every fieldnorm tie, so the pairs are decided by position alone (earliest posting, earliest block)."""
    for seed, n_docs, vocab, lmax in ((3, 3000, 40, 120), (4, 9000, 400, 60), (5, 2000, 7, 30), (6, 40000, 12, 8)):
        c = orc.Corpus.synth(seed, n_docs, vocab, 1, lmax, zipf_s=1.0)
        fn = fieldnorms(orc, c.doc_len)
        for b in (0.75, 0.0):
            oc = orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf, b=b)
            o = oracle_summaries(orc, orc.OracleIndex(oc))
            s = block_summaries(orc, c.post_off, c.post_doc, c.post_tf, fn[c.post_doc], 1.2, b,
                                float(c.doc_len.astype(np.uint64).sum()) / n_docs)
            for key in ("blk_off", "min_doc", "max_doc", "n", "wand_fn", "wand_tf"):
                assert np.array_equal(getattr(s, key), getattr(o, key)), (seed, b, key)
            tok_fn, tok_tf = token_wand(s.blk_off, s.wand_fn, s.wand_tf, s.wand_v)
            assert np.array_equal(tok_fn, o.tok_wand_fn) and np.array_equal(tok_tf, o.tok_wand_tf), (seed, b)
            assert np.array_equal(np.diff(c.post_off.astype(np.int64)), o.df)
            eb = orc.EncodedBlocks(oc)
            nb = eb.n_blocks
            assert np.array_equal(s.min_doc, eb.blk_min[:nb]) and np.array_equal(s.n, eb.blk_n[:nb])
            assert np.array_equal(s.blk_off, eb.term_blk_off)


def test_hand_derived_pairs_and_ties(orc):
    """b = 0: tf() depends on tf alone, every fieldnorm ties.  Term 0: one block, the largest tf (5) at positions 2 and 4 ->
    the first one's norm.  Term 1: 130 postings, tf 3 at positions 1 (block 0) and 128 (block 1): block 0 takes position 1,
    block 1 position 128 (norms 11 and 12), the token the earlier block.  Term 2: no posting -> (255, 0).  Then b = 0.75 on term 0: a larger
    norm lowers tf(), so the shorter document with tf 5 wins even though it comes later."""
    fn = np.array([10, 20, 30, 40, 50] + [7] * 200, np.uint8)
    fn[6], fn[133] = 11, 12
    lists = [([0, 1, 2, 3, 4], [1, 2, 5, 3, 5]),
             (list(range(5, 135)), [1, 3] + [1] * 126 + [3, 2]),
             ([], [])]
    off, doc, tf = _csr(lists)
    s = block_summaries(orc, off, doc, tf, fn[doc], 1.2, 0.0, 10.0)
    assert s.blk_off.tolist() == [0, 1, 3, 3] and s.n.tolist() == [5, 128, 2]
    assert s.min_doc.tolist() == [0, 5, 133] and s.max_doc.tolist() == [4, 132, 134]
    assert s.wand_fn.tolist() == [30, 11, 12] and s.wand_tf.tolist() == [5, 3, 3]
    tok_fn, tok_tf = token_wand(s.blk_off, s.wand_fn, s.wand_tf, s.wand_v)
    assert tok_fn.tolist() == [30, 11, 255] and tok_tf.tolist() == [5, 3, 0]
    # a later block with the same tf() does not replace the earlier one; a strictly larger one does
    assert token_wand([0, 3], [1, 2, 3], [4, 4, 4], [0.5, 0.5, 0.5])[0].tolist() == [1]
    assert token_wand([0, 3], [1, 2, 3], [4, 4, 4], [0.5, 0.5, 0.5 + 2 ** -50])[0].tolist() == [3]
    fn2 = np.array([10, 20, 60, 40, 30] + [7] * 200, np.uint8)
    s = block_summaries(orc, off[:2], doc[:5], tf[:5], fn2[doc[:5]], 1.2, 0.75, 10.0)
    lens = fieldnorm_lengths(orc)
    assert lens[60] > lens[30]
    assert s.wand_fn.tolist() == [30] and s.wand_tf.tolist() == [5]
