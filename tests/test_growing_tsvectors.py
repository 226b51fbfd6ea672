"""CPU-side checks of the growing segment's tsvector calls (bm25x_growing_insert_tsvectors, bm25x_growing_get_new_keys,
bm25x_growing_tsvector_queries): the binding's declarations against include/bm25x.h, and null arguments refused with the
call's name before any device is used."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from util_lib import host_library  # noqa: F401  (host_library: the module fixture m)
from util_tsvector import pack_sorted

ROOT = os.path.dirname(os.path.abspath(__file__)) + "/.."
INSERT, KEYS, QUERIES = "bm25x_growing_insert_tsvectors", "bm25x_growing_get_new_keys", "bm25x_growing_tsvector_queries"
_CTYPES = {"uint32_t": C.c_uint32, "int": C.c_int}


def _bm(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


@pytest.mark.parametrize("name", [INSERT, KEYS, QUERIES])
def test_ctypes_declaration_matches_the_header(m, name):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bm25x.h")).read(), flags=re.S)
    protos = re.findall(rf"\bint\s+({name})\s*\(([^)]*)\)\s*;", hdr)
    assert len(protos) == 1, protos
    params = [" ".join(p.split()) for p in protos[0][1].split(",")]
    argtypes = getattr(m.load_library(), name).argtypes
    assert len(argtypes) == len(params), (params, argtypes)
    for p, a in zip(params, argtypes):
        if "*" in p or "[" in p:
            assert a in (C.c_void_p, C.c_char_p) or issubclass(a, C._Pointer), (p, a)
        else:
            assert a is _CTYPES[p.replace("const ", "").split()[0]], (p, a)


def test_null_arguments(m):
    bm = _bm(m)
    L = m.load_library()
    keep = []
    t = bm._tsvectors(keep, **pack_sorted([{b"alpha": [1, 2]}, {b"beta": [3]}]))
    seed = (C.c_uint8 * 32)()
    seg = C.c_void_p(0x1234)   # never dereferenced: the null checks come first
    for a in ((None, seed, C.byref(t)), (seg, None, C.byref(t)), (seg, seed, None)):
        assert L.bm25x_growing_insert_tsvectors(*a, None) == 1
        assert L.bm25x_last_error().decode() == f"{INSERT}: null argument"
    q_off, q_terms = np.zeros(3, np.uint32), np.zeros(2, np.uint32)
    qo, qt = bm._p(q_off, C.c_uint32), bm._p(q_terms, C.c_uint32)
    for a in ((None, seed, C.byref(t), qo, qt), (seg, None, C.byref(t), qo, qt), (seg, seed, None, qo, qt),
              (seg, seed, C.byref(t), None, qt)):
        assert L.bm25x_growing_tsvector_queries(*a) == 1
        assert L.bm25x_last_error().decode() == f"{QUERIES}: null argument"
    n = C.c_uint32(7)
    keys = np.zeros((1, 16), np.uint8)
    for a in ((None, 1, bm._p(keys, C.c_uint8), C.byref(n)), (seg, 1, bm._p(keys, C.c_uint8), None),
              (seg, 1, None, C.byref(n))):
        assert L.bm25x_growing_get_new_keys(*a) == 1
        assert L.bm25x_last_error().decode() == f"{KEYS}: null argument"
    assert n.value == 7
