"""GPU: the export at full size — C3 of bench.py (10M documents, vocabulary 100k, 128 terms each: ~10M blocks, ~2 GB of
payload, so the encode pass runs in many 256 MiB chunks).  Every output equals the oracle's: the codec's payloads and
directory (orc_encode_blocks), the block and token summaries of its flush restatement (orc_index_build), the norms,
synthetic payloads and Σlen."""
import numpy as np
import pytest

from util_export import oracle_summaries
from util_index import fieldnorms, synthetic_payload
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)

pytestmark = pytest.mark.gpu


def test_export_c3_equals_the_oracle(m, orc):
    c = m.synth_corpus(0xB25C0DE3, 10_000_000, 100_000, 128)
    ix = m.Index.from_corpus(c)
    args, extra = ix.export_blocks()
    ix.close()
    oc = orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf)
    eb = orc.EncodedBlocks(oc)
    nb = eb.n_blocks
    assert eb.n_bytes > 4 * (256 << 20), "C3's payload spans several chunks"
    assert args["data"].tobytes() == eb.bytes[:eb.n_bytes].tobytes(), "payload bytes"
    for key, want in (("term_blk_off", eb.term_blk_off), ("blk_min_doc", eb.blk_min[:nb]), ("blk_n", eb.blk_n[:nb]),
                      ("blk_meta_doc", eb.meta_doc[:nb]), ("blk_meta_tf", eb.meta_tf[:nb]),
                      ("blk_doc_off", eb.doc_off[:nb]), ("blk_tf_off", eb.tf_off[:nb])):
        assert np.array_equal(args[key], want), key
    del eb
    o = oracle_summaries(orc, orc.OracleIndex(oc))
    for key, have, want in (("blk_min_doc", args["blk_min_doc"], o.min_doc), ("blk_max_doc", extra["blk_max_doc"], o.max_doc),
                            ("blk_n", args["blk_n"], o.n), ("blk_wand_fieldnorm", args["blk_wand_fieldnorm"], o.wand_fn),
                            ("blk_wand_tf", args["blk_wand_tf"], o.wand_tf), ("tok_df", extra["tok_df"], o.df),
                            ("tok_wand_fieldnorm", extra["tok_wand_fieldnorm"], o.tok_wand_fn),
                            ("tok_wand_tf", extra["tok_wand_tf"], o.tok_wand_tf)):
        assert np.array_equal(have, want), key
    fn = fieldnorms(orc, c.doc_len)
    total = int(c.doc_len.astype(np.uint64).sum())
    assert np.array_equal(args["doc_fieldnorm"], fn) and args["sum_doc_len"] == total
    assert np.array_equal(args["payload"], synthetic_payload(c.n_docs))
