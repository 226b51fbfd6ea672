"""CPU: the boundary of the mutable growing segment (bm25x_growing_*): its calls are exported, bm25x_growing_info has the
layout the C compiler gives the header, and every call refuses a null handle without touching a device."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from util_lib import host_library  # noqa: F401  (host_library: the module fixture m)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ["bm25x_growing_open", "bm25x_growing_insert", "bm25x_growing_delete", "bm25x_growing_refresh",
         "bm25x_growing_get_info", "bm25x_growing_search_batch", "bm25x_growing_get_index", "bm25x_growing_close"]


def test_growing_segment_symbols_exported(m):
    lib = C.CDLL(os.path.join(ROOT, "vectorchord-bm25_b200", "libbm25x.so"))
    for name in CALLS:
        assert hasattr(lib, name), name


def test_growing_info_layout_matches_the_header(m):
    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    fields = ["n_docs", "n_deleted", "n_postings", "device_bytes", "pending", "device"]
    prog = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "bm25x.h")}"',
            "int main(void) {", 'printf("%zu", sizeof(bm25x_growing_info));']
    prog += [f'printf(" %zu", offsetof(bm25x_growing_info, {f}));' for f in fields]
    prog += ["return 0; }"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-std=c11", "-o", exe, src])
        size, *offs = subprocess.check_output([exe], text=True).split()
    assert C.sizeof(bm.GrowingInfo) == int(size)
    assert [f for f, _ in bm.GrowingInfo._fields_] == fields
    assert [getattr(bm.GrowingInfo, f).offset for f in fields] == [int(o) for o in offs]


def test_null_arguments_refused(m):
    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    L = m.load_library()
    h = C.c_void_p()
    one = np.zeros(4, np.uint32)
    p = one.ctypes.data_as(C.POINTER(C.c_uint32))
    docs = bm._GrowingDocs()
    calls = {
        "bm25x_growing_open": lambda: L.bm25x_growing_open(None, C.byref(h)),
        "bm25x_growing_insert": lambda: L.bm25x_growing_insert(None, C.byref(docs)),
        "bm25x_growing_delete": lambda: L.bm25x_growing_delete(None, 1, p),
        "bm25x_growing_refresh": lambda: L.bm25x_growing_refresh(None),
        "bm25x_growing_get_info": lambda: L.bm25x_growing_get_info(None, C.byref(bm.GrowingInfo())),
        "bm25x_growing_search_batch": lambda: L.bm25x_growing_search_batch(None, 1, p, p, 10, None, None, 0, p, None,
                                                                           None, None, p, None),
        "bm25x_growing_get_index": lambda: L.bm25x_growing_get_index(None, C.byref(bm.IndexLayout()), None),
    }
    for name, call in calls.items():
        assert call() == 1, name
        assert L.bm25x_last_error().decode() == f"{name}: null argument"
    L.bm25x_growing_close(None)  # closing nothing is a no-op
