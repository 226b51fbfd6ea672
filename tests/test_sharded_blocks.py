"""CPU-side checks of the document-sharded index built from stored blocks (bm25x_index_create_sharded_from_blocks): the
blocks are refused with the codes and messages of bm25x_index_create_from_blocks, the shard arguments with those of
bm25x_sharded_create, all before any device is used; without a GPU a well-formed call fails loudly (no CPU fallback);
the ctypes declaration of the binding matches include/bm25x.h."""
import ctypes
import os
import re

import numpy as np
import pytest

from util_lib import host_library, refused  # noqa: F401  (host_library: the module fixture m)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WHO = "bm25x_index_create_from_blocks"


def _corpus(n_docs=600):
    """A small CSR whose term 0 spans three stored blocks (128, 128, 44): term t holds the documents d % (t + 2) == 0."""
    lists = [np.arange(0, n_docs, t + 2, dtype=np.uint32) for t in range(6)]
    off = np.zeros(len(lists) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in lists])
    post_doc = np.concatenate(lists)
    post_tf = (post_doc % 5 + 1).astype(np.uint32)
    doc_len = np.bincount(post_doc, minlength=n_docs).astype(np.uint32) + 1
    return dict(n_docs=n_docs, doc_len=doc_len, n_terms=len(lists), post_off=off, post_doc=post_doc, post_tf=post_tf)


def _blocks(orc, c):
    eb = orc.EncodedBlocks(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"],
                                      c["post_tf"]))
    assert eb.blk_n[0] == 128 and eb.blk_n[1] == 128 and eb.term_blk_off[1] == 3
    return dict(n_docs=c["n_docs"], n_terms=c["n_terms"], term_blk_off=eb.term_blk_off, blk_min_doc=eb.blk_min,
                blk_n=eb.blk_n, blk_meta_doc=eb.meta_doc, blk_meta_tf=eb.meta_tf, blk_doc_off=eb.doc_off,
                blk_tf_off=eb.tf_off, data=eb.bytes[:eb.n_bytes], doc_len=c["doc_len"])


def _host_refusals(orc):
    """(blocks, code, message) of every host refusal of Index.from_blocks; the first three it makes before looking for a
    device, the others after."""
    c = _corpus()
    good = _blocks(orc, c)
    out = []
    for kw in (dict(k1=-1.0), dict(b=1.5)):
        out.append((dict(good, **kw), 1, f"{WHO}: k1/b out of range", True))
    out.append((dict(good, n_docs=0, doc_len=np.zeros(0, np.uint32)), 1, f"{WHO}: empty or malformed corpus", True))
    bad = good["blk_n"].copy()
    bad[0] = 100                                                     # a short block in the middle of a token
    out.append((dict(good, blk_n=bad), 1,
                f"{WHO}: corrupt block directory (block sizes, token ranges or payload offsets)", False))
    bad = good["blk_meta_doc"].copy()
    bad[1] = 33                                                      # bit width 33
    out.append((dict(good, blk_meta_doc=bad), 1,
                f"{WHO}: corrupt block metadata (bitwidth out of bound / unexpected input len)", False))
    bad = good["blk_doc_off"].copy()
    bad[1] = len(good["data"])                                       # payload past the end
    out.append((dict(good, blk_doc_off=bad), 1,
                f"{WHO}: corrupt block directory (block sizes, token ranges or payload offsets)", False))
    bad = good["term_blk_off"].copy()
    bad[0] = 1                                                       # does not run from 0 to n_blocks
    out.append((dict(good, term_blk_off=bad), 1, f"{WHO}: term_blk_off must run from 0 to n_blocks", False))
    return out


def test_block_refusals_match_index_from_blocks(m, orc):
    """The blocks are checked first, whatever the shard arguments, with Index.from_blocks' code and message."""
    gpu = m.device_count() > 0
    for blocks, code, msg, before_device in _host_refusals(orc):
        want = (code, f"bm25x error {code}: {msg}")
        if before_device or gpu:
            assert refused(m, lambda: m.Index.from_blocks(**blocks)) == want
        for n_shards in (1, 2, 0):
            got = refused(m, lambda: m.ShardedIndex.from_blocks(**blocks, n_shards=n_shards))
            assert got == want, (n_shards, got)


@pytest.mark.parametrize("n_shards, bounds", [
    (0, None), (17, None), (16, "small"),
    (2, [1, 300, 600]), (2, [0, 300, 599]), (3, [0, 300, 300, 600]), (3, [0, 350, 300, 600]),
])
def test_shard_refusals_match_sharded_index(m, orc, n_shards, bounds):
    c = _corpus(12) if bounds == "small" else _corpus()
    bounds = None if bounds == "small" else bounds
    if c["n_docs"] == 12:
        # too few postings for the three-block token of _blocks: encode the small corpus directly
        eb = orc.EncodedBlocks(orc.Corpus(c["n_docs"], c["doc_len"], c["n_terms"], c["post_off"], c["post_doc"],
                                          c["post_tf"]))
        blocks = dict(n_docs=12, n_terms=c["n_terms"], term_blk_off=eb.term_blk_off, blk_min_doc=eb.blk_min,
                      blk_n=eb.blk_n, blk_meta_doc=eb.meta_doc, blk_meta_tf=eb.meta_tf, blk_doc_off=eb.doc_off,
                      blk_tf_off=eb.tf_off, data=eb.bytes[:eb.n_bytes], doc_len=c["doc_len"])
    else:
        blocks = _blocks(orc, c)
    want = refused(m, lambda: m.ShardedIndex(**c, n_shards=n_shards, doc_bounds=bounds))
    got = refused(m, lambda: m.ShardedIndex.from_blocks(**blocks, n_shards=n_shards, doc_bounds=bounds))
    assert want[0] == 1 and "bm25x_sharded_create" in want[1]
    assert got == want


def test_no_cpu_fallback(m, orc):
    if m.device_count() > 0:
        pytest.skip("GPU present")
    blocks = _blocks(orc, _corpus())
    code, msg = refused(m, lambda: m.ShardedIndex.from_blocks(**blocks, n_shards=2))
    assert code == 2 and "no CPU fallback" in msg and "bm25x_index_create_sharded_from_blocks" in msg
    code, msg = refused(m, lambda: m.ShardedIndex.from_blocks(**blocks, n_shards=3, doc_bounds=[0, 7, 13, 600],
                                                                devices=[0, 0, 0]))
    assert code == 2 and "no CPU fallback" in msg


_CTYPES = {"uint32_t": ctypes.c_uint32, "int": ctypes.c_int}


def test_ctypes_declaration_matches_the_header(m):
    hdr = open(os.path.join(ROOT, "include", "bm25x.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = re.findall(r"\bint\s+(bm25x_index_create_sharded_from_blocks)\s*\(([^)]*)\)\s*;", hdr)
    assert len(protos) == 1, protos
    name, params = protos[0]
    params = [" ".join(p.split()) for p in params.split(",")]
    assert params[0].startswith("const bm25x_blocks *")
    argtypes = getattr(m.load_library(), name).argtypes
    assert len(argtypes) == len(params), (params, argtypes)
    for p, a in zip(params, argtypes):
        if "*" in p:
            assert a in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(a, ctypes._Pointer), (p, a)
        else:
            assert a is _CTYPES[p.replace("const ", "").split()[0]], (p, a)
