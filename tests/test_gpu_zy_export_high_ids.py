"""GPU: the export of index A of util_sparse (2^32 - 66 documents, ids spread up to 0xFFFFFFFD, built from its stored
blocks): the per-document outputs are skipped (they would be 24 GB); the payloads and directory equal the oracle's
codec byte for byte — the bit-width-32 full block and the byte-width-4 tail above 2^31 included — and the block and token
pairs equal the sparse restatement (util_export over the postings' own norms)."""
from types import SimpleNamespace

import numpy as np
import pytest

from util_export import assert_export_equal, expected_export
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_sparse import B, K1, N_A, T31, full_fieldnorm, high_id_corpus, need, sum_len_of

pytestmark = pytest.mark.gpu


def test_export_index_a(m, orc):
    need(45, 34, "index A (2^32 - 66 documents)")
    c = high_id_corpus(N_A)
    total = sum_len_of(orc, c)
    eb = orc.EncodedBlocks(SimpleNamespace(n_terms=c.n_terms, post_off=c.post_off, post_doc=c.post_doc,
                                           post_tf=c.post_tf))
    fn = full_fieldnorm(c)
    ix = m.Index.from_blocks(c.n_docs, c.n_terms, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf,
                             eb.doc_off, eb.tf_off, eb.bytes[:eb.n_bytes], doc_fieldnorm=fn, sum_doc_len=total, k1=K1, b=B)
    del fn
    got = ix.export_blocks(doc_fieldnorm=False, payload=False)
    ix.close()
    post_fn = c.live_fn[np.searchsorted(c.live, c.post_doc.astype(np.int64))]
    want = expected_export(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, K1, B, None, total, None, post_fn=post_fn)
    assert_export_equal(got, want, "index A")
    (w,) = c.kinds["wide"]
    g = int(got[0]["term_blk_off"][w])
    assert got[0]["blk_meta_doc"][g] == 32 and got[0]["blk_meta_doc"][g + 1] == 0x80 | 4
    assert got[0]["blk_min_doc"][g + 1] >= T31
