"""GPU: a document-sharded index built from stored blocks (bm25x_index_create_sharded_from_blocks) over 2^32 - 66
documents, with a bound at 2^31, a bound inside the bit-width-32 block of the wide term and one inside its byte-width-4
tail, checked bit for bit against the sparse exact reference of tests/util_sparse.py (the corpus and queries of
tests/test_gpu_zy_high_doc_ids.py).  Needs tens of GB of host memory (the norms, and the synthesised payload of the
largest shard); skipped, saying so, when host or device memory is short."""
from types import SimpleNamespace

import numpy as np
import pytest

import _pkg
from test_gpu_zy_high_doc_ids import B, K1, N_A, _Prefix, _need, _queries
from util_sparse import T31, assert_rows, full_fieldnorm, high_id_corpus, reference, sum_len_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.load_library()
    assert mod.device_count() >= 1, "no CUDA device: the engine has no CPU fallback"
    return mod


def test_sharded_from_blocks_above_2_31(m, orc):
    _need(45, 34, "sharded index from blocks (2^32 - 66 documents)")
    c = high_id_corpus(N_A)
    ref = reference(orc, c, K1, B)
    eb = orc.EncodedBlocks(SimpleNamespace(n_terms=c.n_terms, post_off=c.post_off, post_doc=c.post_doc,
                                           post_tf=c.post_tf))
    (w,) = c.kinds["wide"]
    g = int(eb.term_blk_off[w])
    assert eb.meta_doc[g] == 32 and eb.meta_doc[g + 1] == 0x80 | 4
    ids = c.post_doc[int(c.post_off[w]):int(c.post_off[w + 1])].astype(np.int64)
    bounds = np.array(sorted({0, int(ids[64]), T31, int(ids[130]) + 1, N_A}), np.uint32)
    sx = m.ShardedIndex.from_blocks(c.n_docs, c.n_terms, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf,
                                    eb.doc_off, eb.tf_off, eb.bytes[:eb.n_bytes], doc_fieldnorm=full_fieldnorm(c),
                                    sum_doc_len=sum_len_of(orc, c), k1=K1, b=B, n_shards=len(bounds) - 1,
                                    doc_bounds=bounds)
    assert np.array_equal(sx.doc_bounds(), bounds)
    got = sx.search_batch(np.array([0, 1], np.uint32), np.array([w], np.uint32), 1025, want_payload=True)
    assert sorted(got["doc"][0, :int(got["n"][0])].tolist()) == ids.tolist()
    assert_rows(got, ref, [[w]], 1025, "wide term")
    q_off, q_terms, qs = _queries(c, 15)
    pref = _Prefix(ref, 1025)
    for k in (1, 10, 129, 1025):
        res = sx.search_batch(q_off, q_terms, k, want_payload=True)
        assert_rows(res, pref, qs, k, f"sharded from blocks k={k}")
    sx.close()
