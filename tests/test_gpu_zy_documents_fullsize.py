"""GPU: the build from documents at full size.  C3 of bench.py (10M documents, vocabulary 100k, 128 terms each: 1.28G
elements, about 305 chunks) transposed to documents equals Index.from_corpus array for array; and documents up to id
2^32 - 2 (nearly all of them empty) give the posting-side arrays and search rows of the exact sparse reference."""
import numpy as np
import pytest

from util_cuda import download
from util_documents import documents_of_csr
from util_index import LAYOUT, SCALARS, fieldnorms, restate_postings
from util_lib import gpu_library  # noqa: F401  (gpu_library: the module fixture m)
from util_sparse import MAX_N_DOCS, Prefix, SparseReference, assert_rows, high_id_corpus, high_id_queries, need

pytestmark = pytest.mark.gpu

SLICE = 1 << 30


def _same_device_bytes(a_ptr, b_ptr, nbytes, what):
    """[ptr, ptr + nbytes) of two device arrays equal, compared 1 GiB at a time (host memory stays bounded)."""
    for o in range(0, int(nbytes), SLICE):
        n = min(SLICE, int(nbytes) - o)
        assert download(a_ptr + o, n, np.uint8).tobytes() == download(b_ptr + o, n, np.uint8).tobytes(), f"{what} @ {o}"


def test_c3_from_documents_equals_from_corpus(m):
    need(60, 40, "C3 from documents beside C3 from the CSR")
    c = m.synth_corpus(0xB25C0DE3, 10_000_000, 100_000, 128)
    off, term, tf = documents_of_csr(c.n_docs, c.post_off, c.post_doc, c.post_tf)
    got = m.Index.from_documents(off, tf, elem_term=term, n_terms=c.n_terms)
    del off, term, tf
    want = m.Index.from_corpus(c)
    c.free()
    lg, lw = got.layout(), want.layout()
    for name in SCALARS:
        assert getattr(lg, name) == getattr(lw, name), name
    for i, (name, _) in enumerate(LAYOUT):
        assert lg.bytes[i] == lw.bytes[i], name
        _same_device_bytes(lg.dev_ptr[i], lw.dev_ptr[i], lw.bytes[i], name)
    dg, dw = got.derived(), want.derived()
    assert dg.n_champ == dw.n_champ and dg.s1f_min == dw.s1f_min
    for name in ("pdoc", "champ", "champ_off"):
        assert getattr(dg, name + "_bytes") == getattr(dw, name + "_bytes"), name
        _same_device_bytes(getattr(dg, name), getattr(dw, name), getattr(dw, name + "_bytes"), name)
    assert np.array_equal(got.df(), want.df())
    a, w = got.info(), want.info()
    assert [getattr(a, f) for f, _ in type(a)._fields_] == [getattr(w, f) for f, _ in type(w)._fields_]


def test_top_of_the_id_space(m, orc):
    """n_docs = 2^32 - 2: the high-id corpus' documents with postings at their ids (n_docs - 1 included), every other
    document empty (length 0, as the Segment of empty documents has it)."""
    need(90, 34, "documents up to id 2^32 - 2")
    c = high_id_corpus(MAX_N_DOCS)
    order = np.lexsort((np.repeat(np.arange(c.n_terms), np.diff(c.post_off.astype(np.int64))), c.post_doc))
    term = np.repeat(np.arange(c.n_terms, dtype=np.uint32), np.diff(c.post_off.astype(np.int64)))[order]
    tf = c.post_tf[order]
    live, counts = np.unique(c.post_doc, return_counts=True)
    off = np.zeros(c.n_docs + 1, np.uint64)
    off[live.astype(np.int64) + 1] = counts
    np.cumsum(off, out=off)
    ix = m.Index.from_documents(off, tf, elem_term=term, n_terms=c.n_terms)
    del off
    lens = np.zeros(len(live), np.uint64)
    np.add.at(lens, np.searchsorted(live, c.post_doc), c.post_tf.astype(np.uint64))
    live_fn = fieldnorms(orc, lens)
    post_fn = live_fn[np.searchsorted(live, c.post_doc)]
    norms = np.unique(np.append(live_fn, 0))
    lay = ix.layout()
    assert lay.n_docs == MAX_N_DOCS and lay.n_postings == c.post_off[-1] and lay.sum_doc_len == int(lens.sum())
    ref = SparseReference(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, 1.2, 0.75, int(lens.sum()), post_fn=post_fn,
                          norms=norms)
    r = restate_postings(orc, c.n_docs, c.post_off, c.post_doc, c.post_tf, post_fn, norms, 1.2, 0.75, int(lens.sum()))
    for i, (name, dt) in enumerate(LAYOUT):
        if name in ("fieldnorm", "payload"):
            continue
        assert download(lay.dev_ptr[i], lay.bytes[i], dt).tobytes() == getattr(r, name).tobytes(), name
    fn = download(lay.dev_ptr[LAYOUT.index(("fieldnorm", np.uint8))], lay.bytes[9], np.uint8)
    assert np.array_equal(fn[live.astype(np.int64)], live_fn) and np.count_nonzero(fn) == np.count_nonzero(live_fn)
    del fn
    q_off, q_terms, qs = high_id_queries(c, 3)
    pref = Prefix(ref, 1000)
    for k in (1, 10, 100, 1000):
        assert_rows(ix.search_batch(q_off, q_terms, k, want_payload=True), pref, qs, k, f"k={k}")
