"""CPU-side checks of the document-sharded index (bm25x_sharded_*): malformed shard counts, bounds and corpora are refused
before any device is used, with the codes and messages of bm25x_index_create; without a GPU a well-formed call fails
loudly (no CPU fallback); the ctypes declarations of the binding match include/bm25x.h."""
import ctypes
import os
import re

import numpy as np
import pytest

from util_lib import host_library, refused  # noqa: F401  (host_library: the module fixture m)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _corpus(n_docs=40):
    """A small well-formed CSR: term t holds the documents d with d % (t + 2) == 0."""
    lists = [np.arange(0, n_docs, t + 2, dtype=np.uint32) for t in range(6)]
    off = np.zeros(len(lists) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in lists])
    post_doc = np.concatenate(lists)
    post_tf = np.ones(len(post_doc), np.uint32)
    doc_len = np.bincount(post_doc, minlength=n_docs).astype(np.uint32) + 1
    return dict(n_docs=n_docs, doc_len=doc_len, n_terms=len(lists), post_off=off, post_doc=post_doc, post_tf=post_tf)


@pytest.mark.parametrize("n_shards, bounds, what", [
    (0, None, "n_shards=0 must be 1..16"),
    (17, None, "n_shards=17 must be 1..16"),
    (16, "small", "n_docs=12 < n_shards=16"),
    (2, [1, 20, 40], "doc_bounds must ascend strictly from 0 to n_docs=40"),     # does not start at 0
    (2, [0, 20, 39], "doc_bounds must ascend strictly from 0 to n_docs=40"),     # does not end at n_docs
    (3, [0, 20, 20, 40], "doc_bounds must ascend strictly from 0 to n_docs=40"),  # an empty shard
    (3, [0, 25, 20, 40], "doc_bounds must ascend strictly from 0 to n_docs=40"),  # descending
])
def test_malformed_shards_refused(m, n_shards, bounds, what):
    c = _corpus(12) if bounds == "small" else _corpus()
    bounds = None if bounds == "small" else bounds
    code, msg = refused(m, lambda: m.ShardedIndex(**c, n_shards=n_shards, doc_bounds=bounds))
    assert code == 1 and what in msg and "bm25x_sharded_create" in msg, msg


def test_malformed_corpora_refused_as_index_create(m):
    """The corpus checks are bm25x_index_create's, run before the shard checks and before any device is used."""
    cases = []
    c = _corpus()
    c["post_doc"] = c["post_doc"].copy()
    c["post_doc"][[1, 2]] = c["post_doc"][[2, 1]]                        # not ascending inside a term
    cases.append((c, 1, "bm25x_index_create: corrupt corpus (doc ids must be < n_docs and strictly ascending per term, tf != 0)"))
    c = _corpus()
    c["post_tf"] = c["post_tf"].copy()
    c["post_tf"][3] = 0                                                  # tf == 0
    cases.append((c, 1, "bm25x_index_create: corrupt corpus"))
    c = _corpus()
    c["post_doc"] = c["post_doc"].copy()
    c["post_doc"][-1] = 40                                               # doc id >= n_docs
    cases.append((c, 1, "bm25x_index_create: corrupt corpus"))
    c = _corpus()
    c["post_tf"] = c["post_tf"].copy()
    c["post_tf"][0] = 1 << 24                                            # does not fit the packed posting
    cases.append((c, 4, "bm25x_index_create: term frequency >= 2^24 is not supported"))
    for c, code, what in cases:
        for n_shards in (1, 2, 0):   # the corpus is refused first, whatever the shard arguments
            got, msg = refused(m, lambda: m.ShardedIndex(**c, n_shards=n_shards))
            assert got == code and what in msg, (n_shards, msg)


def test_refusals_before_the_device_check_match_index_create(m):
    """Refusals that bm25x_index_create makes before it looks for a device: the same code and the same message."""
    for kw in (dict(k1=-1.0), dict(b=1.5)):
        want = refused(m, lambda: m.Index(**_corpus(), **kw))
        assert want[0] == 1
        assert refused(m, lambda: m.ShardedIndex(**_corpus(), n_shards=2, **kw)) == want
    c = _corpus()
    c["n_docs"], c["doc_len"] = 0, np.zeros(0, np.uint32)
    c["post_doc"] = c["post_doc"][:0]
    c["post_tf"] = c["post_tf"][:0]
    c["post_off"] = np.zeros(len(c["post_off"]), np.uint64)
    want = refused(m, lambda: m.Index(**c))
    assert want[0] == 1 and "empty or malformed corpus" in want[1]
    assert refused(m, lambda: m.ShardedIndex(**c, n_shards=1)) == want


def test_no_cpu_fallback(m):
    if m.device_count() > 0:
        pytest.skip("GPU present")
    code, msg = refused(m, lambda: m.ShardedIndex(**_corpus(), n_shards=2))
    assert code == 2 and "no CPU fallback" in msg
    code, msg = refused(m, lambda: m.ShardedIndex(**_corpus(), n_shards=3, doc_bounds=[0, 7, 13, 40], devices=[0, 0, 0]))
    assert code == 2 and "no CPU fallback" in msg
    code, msg = refused(m, lambda: m.merge_shards([dict(doc=np.zeros((1, 1), np.uint32), score=np.zeros((1, 1), np.float32),
                                                         score64=np.zeros((1, 1)), payload=np.zeros((1, 1, 3), np.uint16),
                                                         n=np.zeros(1, np.uint32))], [0], 1))
    assert code == 2 and "no CPU fallback" in msg


_CTYPES = {"uint32_t": ctypes.c_uint32, "int": ctypes.c_int, "int64_t": ctypes.c_int64}


def test_ctypes_declarations_match_the_header(m):
    """Every bm25x_sharded_* / bm25x_merge_shards prototype of include/bm25x.h against the argtypes the binding declares:
    the same number of parameters, scalars of the same C type, pointers where the header has pointers."""
    hdr = open(os.path.join(ROOT, "include", "bm25x.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = re.findall(r"\b(?:int|void)\s+(bm25x_(?:sharded_[a-z_]+|merge_shards))\s*\(([^)]*)\)\s*;", hdr)
    names = {n for n, _ in protos}
    assert names == {"bm25x_sharded_create", "bm25x_sharded_destroy", "bm25x_sharded_get_info", "bm25x_sharded_set_option",
                     "bm25x_sharded_lookup_terms", "bm25x_sharded_search_batch", "bm25x_sharded_get_shard",
                     "bm25x_merge_shards"}, names
    lib = m.load_library()
    for name, params in protos:
        params = [" ".join(p.split()) for p in params.split(",")]
        argtypes = getattr(lib, name).argtypes
        assert len(argtypes) == len(params), (name, params, argtypes)
        for p, a in zip(params, argtypes):
            if "*" in p:
                assert a in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(a, ctypes._Pointer), (name, p, a)
            else:
                ty = p.replace("const ", "").split()[0]
                assert a is _CTYPES[ty], (name, p, a)
    assert lib.bm25x_sharded_destroy.restype is None
    assert m.MAX_SHARDS == int(re.search(r"#define BM25X_MAX_SHARDS (\d+)", hdr).group(1))
