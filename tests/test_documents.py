"""CPU-side checks of the builds from documents (bm25x_index_create_from_documents and its sharded form): every host
refusal with its code and message, made before any device is used and leaving *out NULL; without a GPU a well-formed call
fails loudly (no CPU fallback); the ctypes mirror of bm25x_documents and the binding's declarations match
include/bm25x.h."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from util_lib import host_library, refused  # noqa: F401  (host_library: the module fixture m)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WHO = "bm25x_index_create_from_documents"


def _docs():
    """Three documents (the second empty) over 6 ordinals, and the same documents keyed."""
    off = np.array([0, 3, 3, 5], np.uint64)
    term = np.array([0, 2, 5, 1, 2], np.uint32)
    tf = np.array([1, 2, 3, 1, 4], np.uint32)
    key = np.zeros((5, 16), np.uint8)
    key[:, 0] = term + 1
    return dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=6), dict(elem_off=off, elem_tf=tf, elem_key=key)


def _refusals():
    """(documents, code, message) of every host refusal."""
    less, keyed = _docs()
    out = []
    bad = dict(less, elem_key=keyed["elem_key"])
    out.append((bad, 1, f"{WHO}: exactly one of elem_key and elem_term must be given"))
    bad = dict(less)
    del bad["elem_term"]
    out.append((bad, 1, f"{WHO}: exactly one of elem_key and elem_term must be given"))
    out.append((dict(keyed, n_terms=4), 1, f"{WHO}: n_terms must be 0 with elem_key (the keys make the vocabulary)"))
    out.append((dict(less, elem_off=np.zeros(1, np.uint64), elem_tf=np.zeros(0, np.uint32),
                     elem_term=np.zeros(0, np.uint32)), 1, f"{WHO}: empty or malformed corpus"))
    out.append((dict(less, k1=-0.5), 1, f"{WHO}: k1/b out of range"))
    out.append((dict(keyed, b=1.01), 1, f"{WHO}: k1/b out of range"))
    out.append((dict(less, elem_off=np.array([1, 3, 3, 5], np.uint64)), 1, f"{WHO}: invalid data: elem_off[0] must be 0"))
    out.append((dict(less, elem_off=np.array([0, 3, 2, 5], np.uint64)), 1,
                f"{WHO}: invalid data: offsets not monotone at document 1"))
    for name, docs in (("keyless", less), ("keyed", keyed)):
        field = "elem_term" if name == "keyless" else "elem_key"
        a = docs[field].copy()
        a[[3, 4]] = a[[4, 3]]                                      # document 2 descending
        out.append((dict(docs, **{field: a}), 1, f"{WHO}: invalid data: keys of document 2 are not strictly ascending"))
        a = docs[field].copy()
        a[1] = a[0]                                                # document 0 repeats a key
        out.append((dict(docs, **{field: a}), 1, f"{WHO}: invalid data: keys of document 0 are not strictly ascending"))
        t = docs["elem_tf"].copy()
        t[4] = 0
        out.append((dict(docs, elem_tf=t), 1, f"{WHO}: invalid data: zero term frequency in document 2"))
        t = docs["elem_tf"].copy()
        t[0] = 1 << 24
        out.append((dict(docs, elem_tf=t), 4,
                    f"{WHO}: term frequency >= 2^24 is not supported by the packed posting layout (document 0)"))
        t = t.copy()
        t[4] = 0                                                   # an invalid document is refused before the tf
        out.append((dict(docs, elem_tf=t), 1, f"{WHO}: invalid data: zero term frequency in document 2"))
    for o in (6, 0xFFFFFFFF):                                     # past n_terms; BM25X_TERM_MISSING
        a = less["elem_term"].copy()
        a[4] = o
        out.append((dict(less, elem_term=a), 1,
                    f"{WHO}: invalid data: a term ordinal of document 2 is not below n_terms=6"))
    a = less["elem_term"].copy()
    a[2] = 7
    t = less["elem_tf"].copy()
    t[4] = 0
    out.append((dict(less, elem_term=a, elem_tf=t), 1,             # the first offending document is named
                f"{WHO}: invalid data: a term ordinal of document 0 is not below n_terms=6"))
    return out


@pytest.mark.parametrize("i", range(len(_refusals())))
def test_host_refusals(m, i):
    docs, code, msg = _refusals()[i]
    want = (code, f"bm25x error {code}: {msg}")
    assert refused(m, lambda: m.Index.from_documents(**docs)) == want
    for n_shards in (1, 2, 0):                                     # the documents first, whatever the shard arguments
        assert refused(m, lambda: m.ShardedIndex.from_documents(**docs, n_shards=n_shards)) == want, n_shards


@pytest.mark.parametrize("n_shards, bounds", [(0, None), (17, None), (4, None), (2, [1, 2, 3]), (2, [0, 2, 2]),
                                              (3, [0, 1, 1, 3]), (2, [0, 3, 3])])
def test_shard_refusals_match_sharded_index(m, n_shards, bounds):
    less, keyed = _docs()
    want = refused(m, lambda: m.ShardedIndex(3, [6, 0, 5], 6, [0, 1, 2, 4, 4, 4, 5], [0, 2, 0, 2, 0],
                                             [1, 1, 2, 4, 3], n_shards=n_shards, doc_bounds=bounds))
    assert want[0] == 1 and "bm25x_sharded_create" in want[1]
    for docs in (less, keyed):
        assert refused(m, lambda: m.ShardedIndex.from_documents(**docs, n_shards=n_shards, doc_bounds=bounds)) == want


def test_null_arguments_leave_out_null(m):
    L = m.load_library()
    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    less, _ = _docs()
    keep = []
    c = bm._documents(keep, less["elem_off"], less["elem_tf"], less["elem_term"], None, less["n_terms"], None, 1.2, 0.75)
    for fn, extra in ((L.bm25x_index_create_from_documents, (0,)),
                      (L.bm25x_index_create_sharded_from_documents, (2, None, None))):
        h = C.c_void_p(0x1234)
        assert fn(None, *extra, C.byref(h)) == 1 and h.value is None
        assert L.bm25x_last_error().decode().endswith(": null argument")
        assert fn(C.byref(c), *extra, None) == 1
        for field in ("elem_off", "elem_tf"):
            cc = bm._Documents.from_buffer_copy(c)
            setattr(cc, field, None)
            h = C.c_void_p(0x1234)
            assert fn(C.byref(cc), *extra, C.byref(h)) == 1 and h.value is None
            assert L.bm25x_last_error().decode() == f"{WHO}: null argument"
        bad = bm._Documents.from_buffer_copy(c)
        bad.k1 = -1.0
        h = C.c_void_p(0x1234)
        assert fn(C.byref(bad), *extra, C.byref(h)) == 1 and h.value is None


def test_no_cpu_fallback(m):
    if m.device_count() > 0:
        pytest.skip("GPU present")
    less, keyed = _docs()
    for docs in (less, keyed):
        code, msg = refused(m, lambda: m.Index.from_documents(**docs))
        assert code == 2 and "no CPU fallback" in msg and WHO in msg
        code, msg = refused(m, lambda: m.ShardedIndex.from_documents(**docs, n_shards=2))
        assert code == 2 and "no CPU fallback" in msg and "bm25x_index_create_sharded_from_documents" in msg


def test_struct_layout_matches_the_header(m):
    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    fields = ["n_docs", "elem_off", "elem_key", "elem_term", "elem_tf", "payload", "n_terms", "k1", "b"]
    prog = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "bm25x.h")}"',
            'int main(void) {', 'printf("%zu", sizeof(bm25x_documents));']
    prog += [f'printf(" %zu", offsetof(bm25x_documents, {f}));' for f in fields]
    prog += ['return 0; }']
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-std=c11", "-o", exe, src])
        size, *offs = subprocess.check_output([exe], text=True).split()
    assert C.sizeof(bm._Documents) == int(size)
    assert [f for f, _ in bm._Documents._fields_] == fields
    assert [getattr(bm._Documents, f).offset for f in fields] == [int(o) for o in offs]


_CTYPES = {"uint32_t": C.c_uint32, "int": C.c_int}


@pytest.mark.parametrize("name", ["bm25x_index_create_from_documents", "bm25x_index_create_sharded_from_documents"])
def test_ctypes_declaration_matches_the_header(m, name):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bm25x.h")).read(), flags=re.S)
    protos = re.findall(rf"\bint\s+({name})\s*\(([^)]*)\)\s*;", hdr)
    assert len(protos) == 1, protos
    params = [" ".join(p.split()) for p in protos[0][1].split(",")]
    assert params[0].startswith("const bm25x_documents *")
    argtypes = getattr(m.load_library(), name).argtypes
    assert len(argtypes) == len(params), (params, argtypes)
    for p, a in zip(params, argtypes):
        if "*" in p:
            assert a in (C.c_void_p, C.c_char_p) or issubclass(a, C._Pointer), (p, a)
        else:
            assert a is _CTYPES[p.replace("const ", "").split()[0]], (p, a)
