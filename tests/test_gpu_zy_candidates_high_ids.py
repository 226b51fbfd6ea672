"""GPU: per-query candidate lists (bm25x_search_candidates, bm25x_search_candidates_sharded) at the top of the 32-bit id
space: an index of n_docs = 2^32 - 2 documents (ids up to 0xFFFFFFFD) from the stored blocks, and the same corpus as a
document-sharded index with bounds at 2^31, 2^31 + 3 and n_docs - 5 (shards of 3 and 5 documents).  Candidate lists hold
the largest ids, the ids around 2^31, holders of the query terms and uniform ids; rows are checked bit for bit against
the sparse exact reference of tests/util_sparse.py restricted to the candidates (no per-query 512 MB bitmap), and the
sharded rows against the unsharded ones.  Each index needs tens of GB of host and device memory; skipped, saying so,
when either is short."""
from types import SimpleNamespace

import numpy as np
import pytest

from util_index import ctid
from util_lib import gpu_library, refused  # noqa: F401  (gpu_library: the module fixture m)
from util_parity import same_rows
from util_sparse import (B, K1, MAX_N_DOCS, T31, assert_rows, full_fieldnorm, high_id_corpus, high_id_queries, need,
                         reference, sum_len_of)

pytestmark = pytest.mark.gpu

KS = (1, 10, 129, 1025, 65535)


class CandidateReference:
    """The sparse reference's full ranking of query i (every document holding a live term) restricted to query i's
    candidates: the ranking is total (score desc, doc asc), so the restriction keeps its order."""

    def __init__(self, ref, qs, lists):
        self.full = [ref.search(q, 1 << 40) for q in qs]
        self.lists = [np.unique(np.asarray(x, np.uint32)) for x in lists]

    def search(self, i, k, allow=None):
        f = self.full[i]
        keep = np.isin(f.doc, self.lists[i])
        d, s = f.doc[keep][:k], f.score64[keep][:k]
        return SimpleNamespace(doc=d, score64=s, score=s.astype(np.float32), payload=ctid(d), n=len(d))


def candidate_lists(rng, c, ref, qs):
    N = c.n_docs
    edges = np.array([N - 1, N - 2, N - 3, T31 - 1, T31, T31 + 1, 0], np.int64)
    lists = []
    for i, q in enumerate(qs):
        held = np.unique(np.concatenate([ref.doc[ref.off[t]:ref.off[t + 1]] for t in ref.live_terms(q)]))
        if i % 5 == 4:
            x = held   # every holder: with k >= |C| the row is the query's whole ranking
        else:
            x = np.concatenate([rng.choice(held, min(len(held), 400), replace=False), edges, edges[:3],
                                rng.integers(0, N, 300), c.live[-2048:][rng.integers(0, 2048, 100)]])
        lists.append(rng.permutation(np.asarray(x, np.int64)))
    return lists


def cand_csr(lists):
    off = np.cumsum([0] + [len(x) for x in lists]).astype(np.uint32)
    return off, np.concatenate([np.asarray(x, np.uint32) for x in lists])


def test_candidates_up_to_the_largest_id(m, orc):
    need(45, 34, "index of 2^32 - 2 documents from blocks")
    c = high_id_corpus(MAX_N_DOCS)
    ref = reference(orc, c, K1, B)
    eb = orc.EncodedBlocks(SimpleNamespace(n_terms=c.n_terms, post_off=c.post_off, post_doc=c.post_doc,
                                           post_tf=c.post_tf))
    blocks = (c.n_docs, c.n_terms, eb.term_blk_off, eb.blk_min, eb.blk_n, eb.meta_doc, eb.meta_tf, eb.doc_off, eb.tf_off,
              eb.bytes[:eb.n_bytes])
    kw = dict(doc_fieldnorm=full_fieldnorm(c), sum_doc_len=sum_len_of(orc, c), k1=K1, b=B)
    q_off, q_terms, qs = high_id_queries(c, 23)
    lists = candidate_lists(np.random.default_rng(29), c, ref, qs)
    assert max(int(x.max()) for x in lists) == MAX_N_DOCS - 1
    c_off, c_docs = cand_csr(lists)
    cref = CandidateReference(ref, qs, lists)
    rows = {}
    ix = m.Index.from_blocks(*blocks, **kw)
    for k in KS:
        rows[k] = ix.search_candidates(q_off, q_terms, c_off, c_docs, k, want_payload=True)
        assert_rows(rows[k], cref, range(len(qs)), k, f"unsharded k={k}")
    # the ids just past the last one: n_docs (0xFFFFFFFE) and 0xFFFFFFFF
    for bad in (MAX_N_DOCS, 0xFFFFFFFF):
        code, msg = refused(m, lambda: ix.search_candidates(q_off[:2], q_terms[:q_off[1]], np.array([0, 2], np.uint32),
                                                             np.array([MAX_N_DOCS - 1, bad], np.uint32), 10))
        assert code == 1 and f"query 0, candidate entry 1: doc id {bad} >= n_docs {MAX_N_DOCS}" in msg, msg
    ix.close()
    bounds = np.array([0, T31, T31 + 3, MAX_N_DOCS - 5, MAX_N_DOCS], np.uint32)
    sx = m.ShardedIndex.from_blocks(*blocks, **kw, n_shards=4, doc_bounds=bounds)
    for k in KS:
        got = sx.search_candidates(q_off, q_terms, c_off, c_docs, k, want_payload=True)
        same_rows({key: got[key] for key in ("doc", "score", "score64", "payload", "n")}, rows[k], f"sharded k={k}")
    code, msg = refused(m, lambda: sx.search_candidates(q_off[:2], q_terms[:q_off[1]], np.array([0, 1], np.uint32),
                                                         np.array([MAX_N_DOCS], np.uint32), 10))
    assert code == 1 and f"doc id {MAX_N_DOCS}" in msg, msg
    sx.close()
