"""CPU: the boundary of the seal (bm25x_growing_seal): the call is exported, bm25x_seal_args has the layout the C compiler
gives the header, null arguments are refused without touching a device; and the restatement of maintain.rs
(util_maintain.maintain) on small cases derived by hand."""
import ctypes as C
import os
import subprocess
import tempfile
from types import SimpleNamespace

import numpy as np

from util_index import ctid
from util_lib import host_library  # noqa: F401  (host_library: the module fixture m)
from util_maintain import MISSING, maintain

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 0xFFFFFFFF


def test_seal_symbol_exported(m):
    lib = C.CDLL(os.path.join(ROOT, "vectorchord-bm25_b200", "libbm25x.so"))
    assert hasattr(lib, "bm25x_growing_seal")


def test_seal_args_layout_matches_the_header(m):
    fields = [f for f, _ in m.SealArgs._fields_]
    assert fields == ["sealed_deleted", "new_keys", "n_new_keys", "sealed_map", "growing_map", "growing_cap", "term_map",
                      "term_cap", "n_growing", "n_source_terms"]
    prog = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "bm25x.h")}"',
            "int main(void) {", 'printf("%zu", sizeof(bm25x_seal_args));']
    prog += [f'printf(" %zu", offsetof(bm25x_seal_args, {f}));' for f in fields]
    prog += ["return 0; }"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-std=c11", "-o", exe, src])
        size, *offs = subprocess.check_output([exe], text=True).split()
    assert C.sizeof(m.SealArgs) == int(size)
    assert [getattr(m.SealArgs, f).offset for f in fields] == [int(o) for o in offs]


def test_seal_null_arguments_refused(m):
    L = m.load_library()
    h = C.c_void_p()
    a = m.SealArgs()
    for call in (lambda: L.bm25x_growing_seal(None, C.byref(a), C.byref(h)),
                 lambda: L.bm25x_growing_seal(C.c_void_p(8), None, C.byref(h)),
                 lambda: L.bm25x_growing_seal(C.c_void_p(8), C.byref(a), None)):
        assert call() == 1
        assert L.bm25x_last_error().decode() == "bm25x_growing_seal: null argument"
    a.n_new_keys = 2  # keys counted, none given
    assert L.bm25x_growing_seal(C.c_void_p(8), C.byref(a), C.byref(h)) == 1
    assert L.bm25x_last_error().decode() == "bm25x_growing_seal: null argument"
    assert not h.value


# ---- the restatement on hand-derived cases ----

def _csr(n_terms, lists):
    """Term-major CSR from {term: [(doc, tf), ...]}."""
    off, doc, tf = [0], [], []
    for t in range(n_terms):
        for d, f in lists.get(t, []):
            doc.append(d)
            tf.append(f)
        off.append(len(doc))
    return np.array(off, np.uint64), np.array(doc, np.uint32), np.array(tf, np.uint32)


def _growing(docs, deleted=None, doc_len=None, payload=None):
    """Growing documents from [[(term, tf), ...], ...]."""
    off = np.cumsum([0] + [len(d) for d in docs]).astype(np.uint64)
    return SimpleNamespace(elem_off=off, elem_term=np.array([t for d in docs for t, _ in d], np.uint32),
                           elem_tf=np.array([f for d in docs for _, f in d], np.uint32),
                           deleted=None if deleted is None else np.array(deleted, np.uint8), doc_len=doc_len,
                           payload=payload)


def test_sealed_length_counts_postings_not_tf():
    """add_element adds 1 per posting (maintain.rs:356-360): a document holding one term at tf 3 has length 1."""
    off, doc, tf = _csr(2, {0: [(0, 3)], 1: [(1, 2)]})
    r = maintain(2, off, doc, tf, _growing([]))
    assert r.doc_len.tolist() == [1, 1]
    assert r.post_doc.tolist() == [0, 1] and r.post_tf.tolist() == [3, 2]
    assert r.payload.tolist() == ctid([0, 1]).tolist()


def test_relabel_order_across_both_segments():
    """Sealed survivors in ascending old id, then growing survivors in ascending ordinal; payloads travel with them,
    the synthetic ones of the OLD id / ordinal."""
    off, doc, tf = _csr(3, {0: [(0, 1), (2, 1), (3, 4)], 1: [(1, 2), (3, 1)], 2: [(2, 5)]})
    g = _growing([[(1, 2)], [(0, 1), (2, 7)], [(0, 3), (MISSING, 4)]], deleted=[0, 1, 0])
    r = maintain(4, off, doc, tf, g, sealed_deleted=[False, True, False, False])
    assert r.sealed_map.tolist() == [0, NONE, 1, 2]
    assert r.growing_map.tolist() == [3, NONE, 4]
    assert r.n_docs == 5 and r.n_terms == 3 and r.term_map.tolist() == [0, 1, 2]
    # term 0: sealed 0, 2, 3 -> 0, 1, 2, then growing ordinal 2 -> 4; term 1: sealed 3 -> 2, growing 0 -> 3; term 2: 2 -> 1
    assert r.post_off.tolist() == [0, 4, 6, 7]
    assert r.post_doc.tolist() == [0, 1, 2, 4, 2, 3, 1]
    assert r.post_tf.tolist() == [1, 1, 4, 3, 1, 2, 5]
    # lengths: sealed by postings (1, 2, 2), growing by Σ tf of every element, the unknown token included (2, 3 + 4)
    assert r.doc_len.tolist() == [1, 2, 2, 2, 7]
    assert r.payload.tolist() == ctid([0, 2, 3]).tolist() + ctid([0, 2]).tolist()


def test_keyed_merge_vanishing_term_and_interleaved_keys():
    """Sealed keys b, d, f; new ordinals 3 -> a, 4 -> e, 5 -> c (never used).  Every posting of d is deleted: d vanishes,
    c has no posting: it never appears.  New order a, b, e, f."""
    key = lambda ch: np.frombuffer(ch.encode() * 16, np.uint8)
    skeys = np.stack([key("b"), key("d"), key("f")])
    nkeys = np.stack([key("a"), key("e"), key("c")])
    off, doc, tf = _csr(3, {0: [(0, 1), (1, 1)], 1: [(1, 2)], 2: [(0, 3)]})
    g = _growing([[(0, 1), (3, 2)], [(4, 1)]], doc_len=np.array([9, 4], np.uint32))
    r = maintain(2, off, doc, tf, g, sealed_deleted=[False, True], sealed_keys=skeys, new_keys=nkeys)
    assert r.term_map.tolist() == [1, MISSING, 3, 0, 2, MISSING]
    assert r.term_keys.tolist() == [key(c).tolist() for c in "abef"]
    assert r.n_terms == 4
    # a: growing 0 (new id 1); b: sealed 0 -> 0, growing 0 -> 1; e: growing 1 -> 2; f: sealed 0 -> 0
    assert r.post_off.tolist() == [0, 1, 3, 4, 5]
    assert r.post_doc.tolist() == [1, 0, 1, 2, 0]
    assert r.post_tf.tolist() == [2, 1, 1, 1, 3]
    assert r.doc_len.tolist() == [2, 9, 4]   # sealed 0 held two postings; growing lengths as stored


def test_keyless_new_ordinals_and_empty_growing_document():
    """An empty growing document survives with length 0 and no posting; ordinals beyond the sealed vocabulary become
    terms, up to the largest one inserted, those without a surviving posting with df 0."""
    off, doc, tf = _csr(2, {0: [(0, 2)]})
    g = _growing([[], [(4, 3)], [(6, 1)]], deleted=[0, 0, 1])
    r = maintain(1, off, doc, tf, g)
    assert r.n_docs == 3 and r.growing_map.tolist() == [1, 2, NONE]
    assert r.doc_len.tolist() == [1, 0, 3]
    assert r.n_terms == 7 and r.term_map.tolist() == list(range(7))
    assert np.diff(r.post_off.astype(np.int64)).tolist() == [1, 0, 0, 0, 1, 0, 0]
    assert r.post_doc.tolist() == [0, 2]
