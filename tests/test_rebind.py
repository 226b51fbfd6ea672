"""CPU: the boundary of the rebind (bm25x_growing_rebind / _sharded): both calls are exported, bm25x_rebind_args has the
layout the C compiler gives the header, the binding's declarations match the prototypes, null arguments are refused
without touching a device; and the restatement of the carried documents (util_rebind) on cases derived by hand."""
import ctypes as C
import os
import re
import subprocess
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest

from util_index import ctid
from util_lib import host_library  # noqa: F401  (host_library: the module fixture m)
from util_maintain import MISSING
from util_rebind import NONE, Refused, late_deleted, restate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("bm25x_growing_rebind", "bm25x_growing_rebind_sharded")


def test_rebind_symbols_exported(m):
    lib = C.CDLL(os.path.join(ROOT, "vectorchord-bm25_b200", "libbm25x.so"))
    for name in CALLS:
        assert hasattr(lib, name), name


def test_rebind_args_layout_matches_the_header(m):
    fields = [f for f, _ in m.RebindArgs._fields_]
    assert fields == ["late_deleted", "n_late_deleted", "n_folded", "n_carried"]
    prog = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "bm25x.h")}"',
            "int main(void) {", 'printf("%zu", sizeof(bm25x_rebind_args));']
    prog += [f'printf(" %zu", offsetof(bm25x_rebind_args, {f}));' for f in fields]
    prog += ["return 0; }"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-std=c11", "-o", exe, src])
        size, *offs = subprocess.check_output([exe], text=True).split()
    assert C.sizeof(m.RebindArgs) == int(size)
    assert [getattr(m.RebindArgs, f).offset for f in fields] == [int(o) for o in offs]


@pytest.mark.parametrize("name", CALLS)
def test_ctypes_declaration_matches_the_header(m, name):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bm25x.h")).read(), flags=re.S)
    protos = re.findall(rf"\bint\s+({name})\s*\(([^)]*)\)\s*;", hdr)
    assert len(protos) == 1, protos
    params = [" ".join(p.split()) for p in protos[0][1].split(",")]
    argtypes = getattr(m.load_library(), name).argtypes
    assert len(argtypes) == len(params) == 3, (params, argtypes)
    for p, a in zip(params, argtypes):
        assert "*" in p and (a is C.c_void_p or issubclass(a, C._Pointer)), (p, a)
    assert argtypes[2]._type_ is m.RebindArgs


@pytest.mark.parametrize("name", CALLS)
def test_null_arguments_refused(m, name):
    L = m.load_library()
    fn = getattr(L, name)
    a = m.RebindArgs()
    a.n_folded = 7
    seg, ix = C.c_void_p(8), C.c_void_p(16)   # never dereferenced: the null checks come first
    for args in ((None, ix, C.byref(a)), (seg, None, C.byref(a)), (seg, ix, None)):
        assert fn(*args) == 1
        assert L.bm25x_last_error().decode() == f"{name}: null argument"
    assert a.n_folded == 7


# ---- the restatement on hand-derived cases ----

def _docs(rows, deleted, payload=None, doc_len=None):
    """Old growing documents from [[(term, tf), ...], ...]."""
    off = np.cumsum([0] + [len(r) for r in rows]).astype(np.uint64)
    return SimpleNamespace(elem_off=off, elem_term=np.array([t for r in rows for t, _ in r], np.uint32),
                           elem_tf=np.array([f for r in rows for _, f in r], np.uint32), deleted=np.array(deleted, np.uint8),
                           payload=payload, doc_len=np.arange(len(rows), dtype=np.uint32) + 10 if doc_len is None else doc_len,
                           doc_fieldnorm=None)


def _rows(r):
    off = r.elem_off.astype(np.int64)
    return [list(zip(r.elem_term[off[i]:off[i + 1]].tolist(), r.elem_tf[off[i]:off[i + 1]].tolist()))
            for i in range(len(off) - 1)]


def test_keyless_ordinals_stay_and_synthetic_ctids_are_the_old_ordinals():
    d = _docs([[(0, 1)], [(2, 2), (9, 1)], [(1, 4), (MISSING, 2)], [(12, 3)]], [0, 1, 0, 1])
    r = restate(d, 2, "keyless")
    assert _rows(r) == [[(1, 4), (MISSING, 2)], []]       # the deleted carried document keeps no element
    assert r.deleted.tolist() == [0, 1]
    assert r.payload.tolist() == ctid([2, 3]).tolist()
    assert r.doc_len.tolist() == [12, 13]
    given = np.arange(12, dtype=np.uint16).reshape(4, 3)
    assert restate(_docs([[], [], [(3, 1)], []], [0] * 4, payload=given), 2, "keyless").payload.tolist() == \
        given[2:].tolist()


def _key(ch):
    return np.frombuffer(ch.encode() * 16, np.uint8)


def test_owned_keys_folded_vanished_and_fresh():
    """Old sealed keys b, d (T = 2); the segment's own keys c (2), a (3), e (4), f (5).  The new index holds a, b, c
    (folded in).  Carried: e and d (the new index lacks them: fresh, ranked d < e), a and b (folded: their new
    ordinals), f only in a deleted carried document (not carried)."""
    old_keys, seg_keys = np.stack([_key("b"), _key("d")]), np.stack([_key(c) for c in "caef"])
    new_keys = np.stack([_key(c) for c in "abc"])
    d = _docs([[(0, 1), (2, 1)], [(3, 2)], [(0, 1), (4, 3)], [(1, 2), (3, 1), (MISSING, 1)], [(5, 1)]],
              [0, 0, 0, 0, 1])
    r = restate(d, 2, "owned", old_keys=old_keys, seg_keys=seg_keys, new_keys=new_keys, new_n_terms=3)
    assert r.owned_keys.tolist() == [_key("d").tolist(), _key("e").tolist()]
    # b -> 1, e -> 3 + 1 = 4; d -> 3, a -> 0
    assert _rows(r) == [[(1, 1), (4, 3)], [(0, 1), (3, 2), (MISSING, 1)], []]


def test_keyed_caller_numbered_translation_and_refusals():
    tmap = np.array([1, MISSING, 0, 2], np.uint32)   # n_source_terms = 4: term 1's key vanished
    ok = _docs([[(1, 1)], [(0, 2), (3, 1)], [(2, 5), (MISSING, 1)]], [0, 0, 0])
    r = restate(ok, 1, "caller", term_map=tmap)
    assert _rows(r) == [[(1, 2), (2, 1)], [(0, 5), (MISSING, 1)]]
    with pytest.raises(Refused, match="growing ordinal 2 holds term ordinal 4 >= n_source_terms=4"):
        restate(_docs([[], [(0, 1)], [(0, 1), (4, 1)], [(1, 1)]], [0] * 4), 1, "caller", term_map=tmap)
    with pytest.raises(Refused, match="growing ordinal 1 holds term ordinal 1, whose key vanished"):
        restate(_docs([[], [(1, 1)], [(9, 1)]], [0] * 3), 1, "caller", term_map=tmap)
    # a deleted carried document is not refused: it keeps no element
    assert _rows(restate(_docs([[], [(1, 1)]], [0, 1]), 1, "caller", term_map=tmap)) == [[]]


def test_late_deletes_through_the_growing_map():
    gmap = np.array([5, NONE, 6, 7], np.uint32)     # ordinal 1 was deleted at the snapshot
    deleted = np.array([0, 1, 1, 1, 1], np.uint8)   # 2 and 3 since; 4 is carried
    assert late_deleted(gmap, deleted).tolist() == [6, 7]
