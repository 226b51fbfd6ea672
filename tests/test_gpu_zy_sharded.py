"""The document-sharded index at full size: BASELINE configs[2] (C3: 10M docs, 128 terms each, 100k 3-term queries, the
bench workload's seeds) in 2 and 4 shards on one GPU against the unsharded index — every output array identical, for
k = 10 and 100.  The whole index and four shards together hold about 31 GB of HBM."""
import numpy as np
import pytest

from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)

pytestmark = pytest.mark.gpu


def test_c3_two_and_four_shards_identical(m):
    c = m.synth_corpus(0xB25C0DE3, 10_000_000, 100_000, 128)
    q_off, q_terms = m.synth_queries(0xB25C0DE3 + 1000, 100_000, 100_000, 3, 3, c.post_off)
    ix = m.Index.from_corpus(c)
    want = {k: ix.search_batch(q_off, q_terms, k, want_payload=True) for k in (10, 100)}
    ix.close()
    for S in (2, 4):
        sx = m.ShardedIndex.from_corpus(c, n_shards=S)
        assert sx.info().n_postings == c.n_postings
        for k in (10, 100):
            got = sx.search_batch(q_off, q_terms, k, want_payload=True)
            assert np.all(got["n"] == k)
            for key in ("doc", "score", "score64", "payload", "n"):
                assert np.array_equal(got[key], want[k][key]), f"C3 S={S} k={k}: `{key}` differs"
            assert got["stats"].postings == want[k]["stats"].postings
            assert got["stats"].queries == want[k]["stats"].queries == 100_000
        sx.close()
