"""CPU: the boundary of the growing segment over a document-sharded index (bm25x_growing_open_sharded,
bm25x_growing_seal_sharded): both calls refuse null arguments without touching a device, without a GPU the binding's
ShardedIndex.growing_segment() fails loudly (no CPU fallback), and the binding declares them as the header does."""
import ctypes
import os
import re

import numpy as np
import pytest

from util_lib import host_library  # noqa: F401  (host_library: the module fixture m)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_null_arguments_refused(m):
    L = m.load_library()
    h = ctypes.c_void_p()
    args = m.SealArgs()
    calls = {
        "bm25x_growing_open_sharded": [lambda: L.bm25x_growing_open_sharded(None, ctypes.byref(h))],
        "bm25x_growing_seal_sharded": [lambda: L.bm25x_growing_seal_sharded(None, ctypes.byref(args), ctypes.byref(h)),
                                       lambda: L.bm25x_growing_seal_sharded(None, None, ctypes.byref(h))],
    }
    for name, fns in calls.items():
        for fn in fns:
            h.value = None
            assert fn() == 1, name
            assert L.bm25x_last_error().decode() == f"{name}: null argument"
            assert not h.value


def test_growing_segment_without_gpu_fails_loudly(m):
    if m.device_count() > 0:
        pytest.skip("GPU present")
    lists = [np.arange(0, 40, t + 2, dtype=np.uint32) for t in range(6)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint64)
    doc = np.concatenate(lists)
    with pytest.raises(m.Bm25xError) as e:
        m.ShardedIndex(40, np.bincount(doc, minlength=40).astype(np.uint32) + 1, len(lists), off, doc,
                       np.ones(len(doc), np.uint32), n_shards=2).growing_segment()
    assert e.value.code == 2 and "no CPU fallback" in str(e.value)


_TYPES = {"bm25x_sharded_index *": ctypes.c_void_p, "bm25x_growing_segment *": ctypes.c_void_p,
          "bm25x_growing_segment **": ctypes.POINTER(ctypes.c_void_p),
          "bm25x_sharded_index **": ctypes.POINTER(ctypes.c_void_p)}


def test_ctypes_declarations_match_the_header(m):
    """The two prototypes of include/bm25x.h against the binding's argtypes, parameter by parameter."""
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bm25x.h")).read(), flags=re.S)
    protos = dict(re.findall(r"\bint\s+(bm25x_growing_(?:open|seal)_sharded)\s*\(([^)]*)\)\s*;", hdr))
    assert set(protos) == {"bm25x_growing_open_sharded", "bm25x_growing_seal_sharded"}, protos
    types = dict(_TYPES, **{"bm25x_seal_args *": ctypes.POINTER(m.SealArgs)})
    lib = m.load_library()
    for name, params in protos.items():
        # "T *name" / "T **name" -> the type with its stars
        want = [types[re.sub(r"\s*(\*+)\s*\w+$", r" \1", " ".join(p.split()))] for p in params.split(",")]
        assert list(getattr(lib, name).argtypes) == want, name
        assert getattr(lib, name).restype is ctypes.c_int
