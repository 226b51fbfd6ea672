"""CPU: the host side of bm25x_evaluate_tsvectors, bm25x_evaluate_batch_sharded and bm25x_evaluate_tsvectors_sharded:
the binding's declarations against include/bm25x.h, and the refusals that come before any handle or device is touched
(null arguments, the tsvectors' host refusals in document then query mode, pair_query, the vectors of the ordinal call)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from util_evaluate_tsvector import SEED, _bm, evaluate_pairs, evaluate_raw
from util_lib import host_library, refused  # noqa: F401  (host_library: the module fixture m)
from util_tsvector import pack_sorted, write_tsvectors

ROOT = os.path.dirname(os.path.abspath(__file__)) + "/.."
NAMES = ["bm25x_evaluate_tsvectors", "bm25x_evaluate_batch_sharded", "bm25x_evaluate_tsvectors_sharded"]
_CTYPES = {"uint32_t": C.c_uint32, "int": C.c_int, "double": C.c_double}
FAKE = C.c_void_p(0x10)   # never dereferenced: every refusal below comes before the handle is read


@pytest.mark.parametrize("name", NAMES)
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


def _good(n=3):
    return pack_sorted([{b"alpha": [1, 2], b"a-lexeme-of-twenty!": [3]}, {}, {b"beta": [4]}][:n])


@pytest.mark.parametrize("sharded", [False, True])
def test_null_arguments(m, sharded):
    bm = _bm(m)
    L = m.load_library()
    fn = L.bm25x_evaluate_tsvectors_sharded if sharded else L.bm25x_evaluate_tsvectors
    who = NAMES[2] if sharded else NAMES[0]
    keep = []
    d, q = bm._tsvectors(keep, **_good()), bm._tsvectors(keep, **_good())
    out = np.zeros(3, np.float64)
    args = [FAKE, bm._seed(SEED), C.byref(d), C.byref(q), None, out.ctypes.data_as(C.POINTER(C.c_double))]
    for i in (0, 1, 2, 3, 5):
        a = list(args)
        a[i] = None
        assert fn(*a) == 1 and L.bm25x_last_error().decode() == f"{who}: null argument", i
    # the ordinal call
    rc, _ = evaluate_pairs(m, None, (np.zeros(2, np.uint32), np.zeros(0), np.zeros(0), np.zeros(2, np.uint32),
                                     np.zeros(0)), sharded=True)
    assert rc == 1 and L.bm25x_last_error().decode() == f"{NAMES[1]}: null argument"


@pytest.mark.parametrize("sharded", [False, True])
def test_host_refusals_in_order(m, sharded):
    """The document tsvectors' refusals (document mode), then the queries' (query mode), then pair_query; out untouched."""
    L = m.load_library()
    who = NAMES[2] if sharded else NAMES[0]
    good = _good()
    no_pos = write_tsvectors([[(b"x", [1])], [(b"y", [1]), (b"z", None)], []])
    bad_off = dict(good, ent_off=np.array([0, 2, 1, 3], np.uint64))
    cases = [(no_pos, good, None, "invalid data: tsvector must have positions (entry 1 of tsvector 1)"),
             (bad_off, bad_off, None, "invalid data: offsets not monotone at tsvector 1"),
             (good, bad_off, None, "invalid data: offsets not monotone at tsvector 1"),
             (good, _good(2), None, "pair_query is NULL, but there are 2 query tsvectors for 3 document tsvectors"),
             (good, _good(2), np.array([0, 2, 1], np.uint32), "pair_query[1] = 2 is not below the 2 query tsvectors")]
    for docs, queries, pq, msg in cases:
        out = np.full(3, 7.0)
        rc, _ = evaluate_raw(m, FAKE, docs, queries, pq, sharded, out=out)
        assert rc == 1 and L.bm25x_last_error().decode() == f"{who}: {msg}", msg
        assert np.all(out == 7.0)
    # a query without positions is no refusal: the call goes on to the handle (a null one here)
    rc, _ = evaluate_raw(m, None, good, no_pos, None, sharded)
    assert rc == 1 and L.bm25x_last_error().decode() == f"{who}: null argument"


def test_ordinal_sharded_vector_refusals(m):
    L = m.load_library()
    off = np.array([0, 2], np.uint32)
    for pairs, msg in (((off, [3, 1], [1, 1], off, [0, 1]), "not strictly ascending"),
                       ((off, [1, 3], [1, 0], off, [0, 1]), "zero term frequency"),
                       ((off, [1, 3], None, off, [0, 1]), "bm25x_evaluate_batch_sharded: null argument")):
        out = np.full(1, 7.0)
        rc, _ = evaluate_pairs(m, FAKE, pairs, sharded=True, out=out)
        assert rc == 1 and msg in L.bm25x_last_error().decode() and out[0] == 7.0


def test_no_cpu_fallback(m):
    """Without a GPU no handle to evaluate on can be built: the builds fail loudly rather than fall back."""
    if m.device_count() > 0:
        pytest.skip("GPU present")
    for fn in (lambda: m.Index.from_tsvectors(SEED, **_good()),
               lambda: m.ShardedIndex.from_tsvectors(SEED, **_good(), n_shards=2)):
        code, msg = refused(m, fn)
        assert code == 2 and "no CPU fallback" in msg
