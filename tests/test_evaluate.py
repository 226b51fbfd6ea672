"""CPU: bm25x_evaluate_batch's host checks, and the fixtures of tests/test_gpu_evaluate.py pinned where no GPU is needed.
- The refusals of bm25x_check_vectors, which evaluate applies to both sides of every pair, and of a null handle.
- The fieldnorm fixture reaches every one of the 256 buckets and both sides of every boundary, and saturates.
- The ulp bound between evaluate and the search, checked between the oracle's evaluate and its exhaustive search over the
  fixture the GPU test compares on: rows at k = 1000 for queries of every term-count class."""
import ctypes as C

import numpy as np

from util_evaluate import (COUNTS, U32_MAX, bucket_lengths, class_queries, exact_corpus, fieldnorm_table, search_pairs,
                           split, sum_tf, ulp_bound, ulps_apart)
from util_lib import host_library, refused  # noqa: F401  (host_library: the module fixture m)


def test_check_vectors_refusals(m):
    ok = ([0, 2, 2, 5], [1, 4, 0, 3, 9], [1, 2, 7, 1, 1])
    m.check_vectors(*ok)
    m.check_vectors(ok[0], ok[1])                                    # a query: no tfs
    m.check_vectors([0], [])                                         # no vectors
    m.check_vectors([0, 0, 0], [])                                   # empty vectors
    cases = {
        "offsets going backwards": (([0, 3, 2, 5], [1, 4, 5, 3, 9], ok[2]), "offsets not monotone at vector 1"),
        "equal ordinals": (([0, 2, 2, 5], [1, 4, 3, 3, 9], ok[2]), "keys of vector 2 are not strictly ascending"),
        "descending ordinals": (([0, 2, 2, 5], [4, 1, 0, 3, 9], ok[2]), "keys of vector 0 are not strictly ascending"),
        "tf = 0": (([0, 2, 2, 5], ok[1], [1, 2, 7, 0, 1]), "zero term frequency in vector 2"),
        "descending query ordinals": (([0, 2, 2, 5], [1, 4, 0, 9, 3], None), "keys of vector 2 are not strictly ascending"),
    }
    for what, (args, msg) in cases.items():
        code, text = refused(m, lambda: m.check_vectors(*args))
        assert code == 1 and msg in text, (what, text)
    L = m.load_library()
    off = np.array([0, 2], np.uint32)
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
    assert L.bm25x_check_vectors(1, None, p(off), None) == 1                       # no offsets
    assert "null argument" in L.bm25x_last_error().decode()
    assert L.bm25x_check_vectors(1, p(off), None, None) == 1                       # elements, but no ordinals
    assert "null argument" in L.bm25x_last_error().decode()
    empty = np.zeros(2, np.uint32)
    assert L.bm25x_check_vectors(1, p(empty), None, None) == 0                     # no elements: no ordinals needed
    assert L.bm25x_check_vectors(0, None, None, None) == 0


def test_evaluate_null_handle(m):
    """A null handle or null arrays are refused on the host, before any device is touched."""
    L = m.load_library()
    off = np.array([0, 1], np.uint32)
    t = np.array([3], np.uint32)
    out = np.full(1, 7.0)
    p = lambda a, ty=C.c_uint32: a.ctypes.data_as(C.POINTER(ty))
    assert L.bm25x_evaluate_batch(None, 1, p(off), p(t), p(t), p(off), p(t), p(out, C.c_double)) == 1
    assert "null argument" in L.bm25x_last_error().decode() and out[0] == 7.0
    assert L.bm25x_evaluate_batch(None, 0, None, None, None, None, None, None) == 1


def test_bucket_fixture_covers_every_bucket_and_both_sides(orc):
    L = orc.lib()
    table = fieldnorm_table(orc)
    assert table[0] == 0 and np.all(np.diff(table) > 0)
    cases = bucket_lengths(orc)
    lengths = {n for n, _ in cases}
    for n, tfs in cases:
        assert sum_tf(tfs) == n and all(1 <= t <= U32_MAX for t in tfs) and len(tfs) <= 3
    norms = {L.orc_length_to_fieldnorm(n) for n in lengths}
    assert norms == set(range(256))
    for f in range(1, 256):                      # both sides of every boundary
        below, at = int(table[f]) - 1, int(table[f])
        assert below in lengths and at in lengths and at + 1 in lengths
        assert L.orc_length_to_fieldnorm(below) == f - 1 and L.orc_length_to_fieldnorm(at) == f
    assert U32_MAX in lengths and L.orc_length_to_fieldnorm(U32_MAX) == 255
    assert any(sum(int(t) for t in tfs) > U32_MAX for _, tfs in cases)         # the Σ saturates
    assert split(0) == [] and split(2) == [2] and split(10) == [3, 4, 3]


def test_ulp_bound_of_evaluate_against_search_on_the_oracle(orc):
    """The bound tests/test_gpu_evaluate.py demands of the GPU, between orc_evaluate and orc_search_exhaustive (which the
    GPU paths equal bit for bit): every row at k = 1000 of queries of every term-count class, the document restated
    doc-major.  The two differ in the last bits on some rows; the bound must hold on all."""
    n_docs, doc_len, T, off, doc, tf = exact_corpus(5)
    c = orc.Corpus(n_docs, doc_len, T, off, doc, tf)
    oix = orc.OracleIndex(c)
    q_off, q_terms = class_queries(6, T)
    nq, k = len(q_off) - 1, 1000
    rows_doc = np.zeros((nq, k), np.uint32)
    rows_n = np.zeros(nq, np.uint32)
    scores = []
    for i in range(nq):
        d, s, _ = oix.search_exhaustive(q_terms[q_off[i]:q_off[i + 1]], k)
        rows_doc[i, :len(d)], rows_n[i] = d, len(d)
        scores.append(s)
    assert np.count_nonzero(rows_n == k) >= len(COUNTS)
    d_off, d_terms, d_tfs, p_off, p_terms, matched, qi = search_pairs(n_docs, off, doc, tf, q_off, q_terms, rows_doc,
                                                                    rows_n)
    L = orc.lib()
    ev = np.array([oix.evaluate(d_terms[d_off[p]:d_off[p + 1]], d_tfs[d_off[p]:d_off[p + 1]],
                                p_terms[p_off[p]:p_off[p + 1]]) for p in range(len(qi))])
    se = np.concatenate(scores)
    assert len(ev) == len(se) > 19000 and np.all(matched >= 1)
    # the restated documents have the index's exact lengths, so evaluate sees the norms the search scores with
    ids = np.concatenate([rows_doc[i, :rows_n[i]] for i in range(nq)])
    lens = np.add.reduceat(d_tfs.astype(np.int64), d_off[:-1].astype(np.int64))
    assert np.array_equal(lens, doc_len[ids].astype(np.int64))
    assert all(L.orc_length_to_fieldnorm(int(doc_len[d])) == L.orc_index_fieldnorm(oix.h, int(d)) for d in ids[::97])
    apart = ulps_apart(ev, se)
    bound = np.array([ulp_bound(int(x)) for x in matched])
    assert np.all(apart <= bound), np.max(apart - bound)
    assert np.count_nonzero(apart) > 100          # the two orders do differ: the test compares something
