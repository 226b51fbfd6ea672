"""CPU-side checks of the tsvector entry points (bm25x_cast_tsvectors, bm25x_index_create_from_tsvectors,
bm25x_tsvector_queries): the ctypes mirror of bm25x_tsvectors and the binding's declarations against include/bm25x.h,
every host refusal with its code and message before any device is used, and the restated casts of the golden passages."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from util_lib import host_library, refused  # noqa: F401  (host_library: the module fixture m)
from util_tsvector import cast, pack_sorted, write_tsvectors

ROOT = os.path.dirname(os.path.abspath(__file__)) + "/.."
SEED = bytes(range(32))
CAST, BUILD, QUERIES = "bm25x_cast_tsvectors", "bm25x_index_create_from_tsvectors", "bm25x_tsvector_queries"


def _bm(m):
    return __import__(m.__name__ + ".bm25x", fromlist=["x"])


def _good():
    return pack_sorted([{b"alpha": [1, 2], b"a-lexeme-of-twenty!": [3]}, {}, {b"beta": [4]}])


def _refusals():
    """(tsvectors, document-mode message, query-mode message or None when the query cast accepts them)."""
    out = []
    t = _good()
    out.append((dict(t, ent_off=np.array([1, 2, 2, 3], np.uint64)),
                "invalid data: ent_off[0] and byte_off[0] must be 0", "same"))
    out.append((dict(t, byte_off=np.array([2, 20, 20, 30], np.uint64)),
                "invalid data: ent_off[0] and byte_off[0] must be 0", "same"))
    out.append((dict(t, ent_off=np.array([0, 2, 1, 3], np.uint64)), "invalid data: offsets not monotone at tsvector 1",
                "same"))
    bo = t["byte_off"].copy()
    bo[2] = bo[1] - 1
    out.append((dict(t, byte_off=bo), "invalid data: offsets not monotone at tsvector 1", "same"))
    # lexeme past the area: entry 0 of vector 2 claims 200 bytes
    e = t["entries"].copy()
    e[2] = (e[2] & ~np.uint32(0xFFE)) | np.uint32(200 << 1)
    out.append((dict(t, entries=e), "invalid data: the lexeme of entry 0 of tsvector 2 runs past its area", "same"))
    # count past the area: the last vector's area cut just before its count
    bo = t["byte_off"].copy()
    bo[3] = bo[2] + 5
    d = t["data"][:int(bo[3])]
    out.append((dict(t, byte_off=bo, data=d),
                "invalid data: the position count of entry 0 of tsvector 2 runs past its area", "same"))
    # no positions: fine for a query, refused for a document
    nopos = write_tsvectors([[(b"x", [1])], [(b"y", [1]), (b"z", None)]])
    out.append((nopos, "invalid data: tsvector must have positions (entry 1 of tsvector 1)", None))
    # the first offending vector is named
    e = t["entries"].copy()
    e[1] = (e[1] & ~np.uint32(0xFFE)) | np.uint32(2000 << 1)
    e[2] = (e[2] & ~np.uint32(0xFFE)) | np.uint32(2000 << 1)
    out.append((dict(t, entries=e), "invalid data: the lexeme of entry 1 of tsvector 0 runs past its area", "same"))
    return out


@pytest.mark.parametrize("i", range(len(_refusals())))
def test_host_refusals(m, i):
    tsv, doc_msg, query_msg = _refusals()[i]
    bm = _bm(m)
    for who, as_query in ((CAST, False), (CAST, True)):
        msg = doc_msg if not as_query else (doc_msg if query_msg == "same" else None)
        if msg is None:
            continue
        want = (1, f"bm25x error 1: {who}: {msg}")
        assert refused(m, lambda: bm.cast_tsvectors(SEED, **tsv, as_query=as_query)) == want
    want = (1, f"bm25x error 1: {BUILD}: {doc_msg}")
    assert refused(m, lambda: m.Index.from_tsvectors(SEED, **tsv)) == want


def test_build_refuses_check_common(m):
    t = _good()
    empty = dict(ent_off=np.zeros(1, np.uint64), entries=np.zeros(0, np.uint32), byte_off=np.zeros(1, np.uint64),
                 data=np.zeros(0, np.uint8))
    for tsv, kw, msg in ((empty, {}, "empty or malformed corpus"), (t, dict(k1=-1.0), "k1/b out of range"),
                         (t, dict(b=1.5), "k1/b out of range"), (t, dict(b=float("nan")), "k1/b out of range")):
        assert refused(m, lambda: m.Index.from_tsvectors(SEED, **tsv, **kw)) == (1, f"bm25x error 1: {BUILD}: {msg}")
    # the tsvectors are checked first
    bad = dict(t, ent_off=np.array([0, 2, 1, 3], np.uint64))
    assert refused(m, lambda: m.Index.from_tsvectors(SEED, **bad, k1=-1.0))[1].endswith("offsets not monotone at tsvector 1")


def test_null_arguments(m):
    bm = _bm(m)
    L = m.load_library()
    keep = []
    t = bm._tsvectors(keep, **_good())
    seed = (C.c_uint8 * 32)()
    off = np.zeros(4, np.uint64)
    key = np.zeros((3, 16), np.uint8)
    tf = np.zeros(3, np.uint32)
    args = (C.byref(t), seed, 0, 0, bm._p(off, C.c_uint64), bm._p(key, C.c_uint8), bm._p(tf, C.c_uint32))
    for i in (0, 1, 4, 5, 6):
        a = list(args)
        a[i] = None
        assert L.bm25x_cast_tsvectors(*a) == 1
        assert L.bm25x_last_error().decode() == f"{CAST}: null argument"
    a = list(args)
    a[6] = None
    a[2] = 1                                                       # query mode: out_tf may be NULL
    assert L.bm25x_cast_tsvectors(*a) != 1 or "null" not in L.bm25x_last_error().decode()
    for field in ("ent_off", "byte_off", "entries", "bytes"):
        tt = bm._Tsvectors.from_buffer_copy(t)
        setattr(tt, field, None)
        assert L.bm25x_cast_tsvectors(C.byref(tt), *args[1:]) == 1
        assert L.bm25x_last_error().decode() == f"{CAST}: null argument", field
    h = C.c_void_p(0x1234)
    for a in ((None, seed), (C.byref(t), None)):
        h = C.c_void_p(0x1234)
        assert L.bm25x_index_create_from_tsvectors(a[0], a[1], None, 1.2, 0.75, 0, C.byref(h)) == 1 and h.value is None
        assert L.bm25x_last_error().decode() == f"{BUILD}: null argument"
    assert L.bm25x_index_create_from_tsvectors(C.byref(t), seed, None, 1.2, 0.75, 0, None) == 1
    q_off = np.zeros(4, np.uint32)
    q_terms = np.zeros(3, np.uint32)
    for a in ((None, seed, C.byref(t)), (C.c_void_p(0x1), None, C.byref(t)), (C.c_void_p(0x1), seed, None)):
        assert L.bm25x_tsvector_queries(*a, bm._p(q_off, C.c_uint32), bm._p(q_terms, C.c_uint32)) == 1
        assert L.bm25x_last_error().decode() == f"{QUERIES}: null argument"


def test_no_cpu_fallback(m):
    if m.device_count() > 0:
        pytest.skip("GPU present")
    bm = _bm(m)
    for fn, who in ((lambda: bm.cast_tsvectors(SEED, **_good()), CAST),
                    (lambda: bm.cast_tsvectors(SEED, **_good(), as_query=True), CAST),
                    (lambda: m.Index.from_tsvectors(SEED, **_good()), BUILD)):
        code, msg = refused(m, fn)
        assert code == 2 and "no CPU fallback" in msg and who in msg


def test_struct_layout_matches_the_header(m):
    bm = _bm(m)
    fields = ["n", "ent_off", "entries", "byte_off", "bytes"]
    prog = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "bm25x.h")}"',
            'int main(void) {', 'printf("%zu", sizeof(bm25x_tsvectors));']
    prog += [f'printf(" %zu", offsetof(bm25x_tsvectors, {f}));' for f in fields]
    prog += ['return 0; }']
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-std=c11", "-o", exe, src])
        size, *offs = subprocess.check_output([exe], text=True).split()
    assert C.sizeof(bm._Tsvectors) == int(size)
    assert [f for f, _ in bm._Tsvectors._fields_] == fields
    assert [getattr(bm._Tsvectors, f).offset for f in fields] == [int(o) for o in offs]


_CTYPES = {"uint32_t": C.c_uint32, "int": C.c_int, "double": C.c_double}


@pytest.mark.parametrize("name", [CAST, BUILD, QUERIES])
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


def _golden_tsvectors(golden):
    """The golden passages as tsvectors: each lexeme with the positions where it occurs (1-based)."""
    docs = []
    for lex in golden["doc_lexemes"]:
        d = {}
        for p, w in enumerate(lex, 1):
            d.setdefault(w.encode(), []).append(p)
        docs.append(d)
    return pack_sorted(docs)


def test_golden_restated_cast_lengths(m, golden):
    off, keys, tf = cast(_bm(m).intern, SEED, _golden_tsvectors(golden))
    lengths = np.add.reduceat(tf.astype(np.int64), off[:-1].astype(np.int64))
    assert lengths.tolist() == golden["doc_lengths"]
    for i in range(len(off) - 1):                                  # each row ascending bytewise and distinct
        row = [bytes(k) for k in keys[off[i]:off[i + 1]]]
        assert row == sorted(set(row))
    qo, qk, qt = cast(_bm(m).intern, SEED, _golden_tsvectors(golden), as_query=True)
    assert qt is None and np.array_equal(qo, off) and np.array_equal(qk, keys)
