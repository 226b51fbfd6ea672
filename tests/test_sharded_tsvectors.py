"""CPU-side checks of the sharded build from tsvectors (bm25x_index_create_sharded_from_tsvectors) and the query cast of a
sharded index (bm25x_tsvector_queries_sharded): every host refusal with its code and message, in order, before any
device is used; null arguments; no CPU fallback; the binding's declarations against include/bm25x.h."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from util_lib import host_library, refused  # noqa: F401  (host_library: the module fixture m)
from util_tsvector import pack_sorted, write_tsvectors

ROOT = os.path.dirname(os.path.abspath(__file__)) + "/.."
SEED = bytes(range(32))
BUILD, QUERIES = "bm25x_index_create_sharded_from_tsvectors", "bm25x_tsvector_queries_sharded"


def _bm(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


def _good():
    return pack_sorted([{b"alpha": [1, 2], b"a-lexeme-of-twenty!": [3]}, {}, {b"beta": [4]}])


def _tsvector_refusals():
    """(tsvectors, message) of bm25x_index_create_from_tsvectors' host refusals of a document batch."""
    t = _good()
    out = [(dict(t, ent_off=np.array([1, 2, 2, 3], np.uint64)), "invalid data: ent_off[0] and byte_off[0] must be 0"),
           (dict(t, ent_off=np.array([0, 2, 1, 3], np.uint64)), "invalid data: offsets not monotone at tsvector 1")]
    e = t["entries"].copy()
    e[2] = (e[2] & ~np.uint32(0xFFE)) | np.uint32(200 << 1)
    out.append((dict(t, entries=e), "invalid data: the lexeme of entry 0 of tsvector 2 runs past its area"))
    bo = t["byte_off"].copy()
    bo[3] = bo[2] + 5
    out.append((dict(t, byte_off=bo, data=t["data"][:int(bo[3])]),
                "invalid data: the position count of entry 0 of tsvector 2 runs past its area"))
    out.append((write_tsvectors([[(b"x", [1])], [(b"y", [1]), (b"z", None)]]),
                "invalid data: tsvector must have positions (entry 1 of tsvector 1)"))
    return out


@pytest.mark.parametrize("i", range(len(_tsvector_refusals())))
def test_tsvector_refusals(m, i):
    tsv, msg = _tsvector_refusals()[i]
    want = (1, f"bm25x error 1: {BUILD}: {msg}")
    assert refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **tsv)) == want
    # before the build's arguments and the shard arguments
    assert refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **tsv, k1=-1.0, n_shards=0)) == want


def test_check_common_refusals(m):
    t = _good()
    empty = dict(ent_off=np.zeros(1, np.uint64), entries=np.zeros(0, np.uint32), byte_off=np.zeros(1, np.uint64),
                 data=np.zeros(0, np.uint8))
    for tsv, kw, msg in ((empty, {}, "empty or malformed corpus"), (t, dict(k1=-1.0), "k1/b out of range"),
                         (t, dict(b=1.5), "k1/b out of range"), (t, dict(b=float("nan")), "k1/b out of range"),
                         (t, dict(k1=float("nan"), n_shards=0), "k1/b out of range")):   # before the shard arguments
        got = refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **tsv, **kw))
        assert got == (1, f"bm25x error 1: {BUILD}: {msg}"), kw


def test_shard_argument_refusals(m):
    t = _good()   # 3 tsvectors
    for kw, msg in ((dict(n_shards=0), "n_shards=0 must be 1..16"), (dict(n_shards=17), "n_shards=17 must be 1..16"),
                    (dict(n_shards=4), "n_docs=3 < n_shards=4 (every shard holds at least one document)"),
                    (dict(n_shards=2, doc_bounds=[0, 0, 3]), "doc_bounds must ascend strictly from 0 to n_docs=3"),
                    (dict(n_shards=2, doc_bounds=[1, 2, 3]), "doc_bounds must ascend strictly from 0 to n_docs=3"),
                    (dict(n_shards=2, doc_bounds=[0, 2, 4]), "doc_bounds must ascend strictly from 0 to n_docs=3"),
                    (dict(n_shards=3, doc_bounds=[0, 2, 1, 3]), "doc_bounds must ascend strictly from 0 to n_docs=3")):
        got = refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **t, **kw))
        assert got == (1, f"bm25x error 1: bm25x_sharded_create: {msg}"), kw


def test_null_arguments(m):
    bm = _bm(m)
    L = m.load_library()
    keep = []
    t = bm._tsvectors(keep, **_good())
    seed = (C.c_uint8 * 32)()
    for a in ((None, seed), (C.byref(t), None)):
        h = C.c_void_p(0x1234)
        assert L.bm25x_index_create_sharded_from_tsvectors(a[0], a[1], None, 1.2, 0.75, 2, None, None, C.byref(h)) == 1
        assert h.value is None and L.bm25x_last_error().decode() == f"{BUILD}: null argument"
    assert L.bm25x_index_create_sharded_from_tsvectors(C.byref(t), seed, None, 1.2, 0.75, 2, None, None, None) == 1
    assert L.bm25x_last_error().decode() == f"{BUILD}: null argument"
    for field in ("ent_off", "byte_off", "entries", "bytes"):
        tt = bm._Tsvectors.from_buffer_copy(t)
        setattr(tt, field, None)
        h = C.c_void_p(0x1234)
        assert L.bm25x_index_create_sharded_from_tsvectors(C.byref(tt), seed, None, 1.2, 0.75, 2, None, None,
                                                           C.byref(h)) == 1
        assert h.value is None and L.bm25x_last_error().decode() == f"{BUILD}: null argument", field
    q_off = np.zeros(4, np.uint32)
    q_terms = np.zeros(3, np.uint32)
    for a in ((None, seed, C.byref(t)), (C.c_void_p(0x1), None, C.byref(t)), (C.c_void_p(0x1), seed, None)):
        assert L.bm25x_tsvector_queries_sharded(*a, bm._p(q_off, C.c_uint32), bm._p(q_terms, C.c_uint32)) == 1
        assert L.bm25x_last_error().decode() == f"{QUERIES}: null argument"
    assert L.bm25x_tsvector_queries_sharded(C.c_void_p(0x1), seed, C.byref(t), None, bm._p(q_terms, C.c_uint32)) == 1
    assert L.bm25x_last_error().decode() == f"{QUERIES}: null argument"


def test_no_cpu_fallback(m):
    if m.device_count() > 0:
        pytest.skip("GPU present")
    for kw in ({}, dict(n_shards=3, doc_bounds=[0, 1, 2, 3]), dict(n_shards=2, devices=[0, 0])):
        code, msg = refused(m, lambda: m.ShardedIndex.from_tsvectors(SEED, **_good(), **kw))
        assert code == 2 and "no CPU fallback" in msg and BUILD in msg, kw


_CTYPES = {"uint32_t": C.c_uint32, "int": C.c_int, "double": C.c_double}


@pytest.mark.parametrize("name", [BUILD, QUERIES])
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
