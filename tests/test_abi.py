"""CPU-side checks of the boundary: the C-ABI library loads and exports every symbol include/bm25x.h declares,
the host logic fails loudly without a GPU (no CPU fallback), and the product's synthetic generator agrees
bit for bit with the oracle's independent restatement of the same spec."""
import ctypes
import os
import re

import numpy as np
import pytest

import _pkg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def m():
    mod = _pkg.load()
    mod.build_library()
    mod.load_library()
    return mod


def test_exports_every_declared_symbol(m):
    hdr = "".join(open(os.path.join(ROOT, "include", f)).read() for f in sorted(os.listdir(os.path.join(ROOT, "include")))
                  if f.endswith(".h"))
    names = set(re.findall(r"\b(bm25x_[a-z_0-9]+)\s*\(", hdr)) - {"bm25x_broker_backend"}  # (a function-pointer typedef)
    assert len(names) >= 20
    lib = ctypes.CDLL(os.path.join(ROOT, "vectorchord-bm25_b200", "libbm25x.so"))
    for n in sorted(names):
        assert hasattr(lib, n), f"{n} declared in include/*.h but not exported"


def test_library_has_only_sm90a_code(m):
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", os.path.join(ROOT, "vectorchord-bm25_b200", "libbm25x.so")],
                         capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_no_cpu_fallback(m):
    if m.device_count() > 0:
        pytest.skip("GPU present")
    c = m.synth_corpus(1, 100, 50, 8)
    with pytest.raises(m.Bm25xError) as e:
        m.Index.from_corpus(c)
    assert e.value.code == 2 and "no CPU fallback" in str(e.value)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "vectorchord-bm25_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".h", ".cuh", "Makefile")):
                assert "oracle" not in open(os.path.join(dp, f)).read().lower().replace(
                    "the oracle (oracle/bm25_oracle.c) restates the same spec independently; tests compare the two.", ""), f


@pytest.mark.parametrize("cfg", [dict(seed=0xB25C0DE1, n=1000, vocab=1000, lmin=32, lmax=32, zipf=0.0),
                                 dict(seed=5, n=4000, vocab=700, lmin=1, lmax=150, zipf=1.0),
                                 dict(seed=6, n=2500, vocab=40, lmin=0, lmax=20, zipf=0.7)])
def test_synth_matches_oracle_generator(m, orc, cfg):
    a = m.synth_corpus(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"], nthreads=3)
    b = orc.Corpus.synth(cfg["seed"], cfg["n"], cfg["vocab"], cfg["lmin"], cfg["lmax"], cfg["zipf"])
    for x in ("doc_len", "post_off", "post_doc", "post_tf"):
        assert np.array_equal(getattr(a, x), getattr(b, x)), x
    ix = orc.OracleIndex(b)
    qa = m.synth_queries(cfg["seed"] + 1000, 64, cfg["vocab"], 1, 8, a.post_off, cfg["zipf"])
    qb = orc.gen_queries(cfg["seed"] + 1000, 64, cfg["vocab"], 1, 8, ix.df, cfg["zipf"])
    assert np.array_equal(qa[0], qb[0]) and np.array_equal(qa[1], qb[1])
    # spec properties: Σ tf = doc length; doc ids ascend inside a term
    assert int(a.post_tf.astype(np.uint64).sum()) == int(a.doc_len.astype(np.uint64).sum())
    for t in range(min(cfg["vocab"], 50)):
        seg = a.post_doc[a.post_off[t]:a.post_off[t + 1]]
        assert np.all(np.diff(seg.astype(np.int64)) > 0)


def test_document_query_types(m):
    m.Document([1, 5, 9], [1, 2, 3])
    with pytest.raises(ValueError):
        m.Document([5, 1], [1, 1])      # not ascending (vector.rs:56-66)
    with pytest.raises(ValueError):
        m.Document([1, 2], [1, 0])      # tf == 0
    with pytest.raises(ValueError):
        m.Query([3, 3])


def test_struct_layouts_match_the_header(m):
    """The ctypes mirrors in bm25x.py (the stand-in for the Rust #[repr(C)] structs of INTEGRATION.md) must have the
    sizes and field offsets the C compiler gives include/bm25x.h."""
    import ctypes as C
    import subprocess
    import tempfile

    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    HEADER = os.path.join(ROOT, "include", "bm25x.h")
    structs = {"bm25x_corpus": (bm._Corpus, ["n_docs", "doc_len", "payload", "n_terms", "term_key", "post_off",
                                             "post_doc", "post_tf", "k1", "b"]),
               "bm25x_blocks": (bm._Blocks, ["n_docs", "doc_len", "doc_fieldnorm", "sum_doc_len", "payload", "n_terms",
                                             "term_key", "term_blk_off", "n_blocks", "blk_min_doc", "blk_n",
                                             "blk_meta_doc", "blk_meta_tf", "blk_doc_off", "blk_tf_off", "bytes",
                                             "n_bytes", "k1", "b", "blk_wand_fieldnorm", "blk_wand_tf"]),
               "bm25x_index_info": (bm.IndexInfo, ["n_docs", "n_terms", "n_postings", "sum_doc_len", "avgdl", "k1", "b",
                                                   "device_bytes", "n_blocks", "device"]),
               "bm25x_index_layout": (bm.IndexLayout, ["n_docs", "n_terms", "n_postings", "n_postings_padded",
                                                       "n_blocks", "sum_doc_len", "k1", "b", "avgdl", "dev_ptr",
                                                       "bytes", "device"]),
               "bm25x_index_derived": (bm.IndexDerived, ["pdoc", "pdoc_bytes", "champ", "champ_bytes", "champ_off",
                                                         "champ_off_bytes", "n_champ", "s1f_min", "device"]),
               "bm25x_search_stats": (bm.SearchStats, ["kernel_ms", "h2d_ms", "d2h_ms", "postings", "bytes_algo",
                                                       "launches", "queries", "postings_fetched"])}
    prog = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', 'int main(void) {']
    for cname, (_, fields) in structs.items():
        prog.append(f'printf("{cname} %zu", sizeof({cname}));')
        for f in fields:
            prog.append(f'printf(" %zu", offsetof({cname}, {f}));')
        prog.append('printf("\\n");')
    prog.append('return 0; }')
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(src, "w").write("\n".join(prog))
        subprocess.check_call(["gcc", "-std=c11", "-o", exe, src])
        out = subprocess.check_output([exe], text=True)
    for line in out.splitlines():
        name, size, *offs = line.split()
        cls, fields = structs[name]
        assert C.sizeof(cls) == int(size), f"{name}: ctypes size {C.sizeof(cls)} != C {size}"
        assert [f for f, _ in cls._fields_] == fields, f"{name}: field order"
        assert [getattr(cls, f).offset for f in fields] == [int(o) for o in offs], f"{name}: field offsets"


def test_vector_invariants_in_c(m):
    """bm25x_check_vectors = what Document::new / Query::new enforce (crates/bm25/src/vector.rs:46-134): strictly ascending
    keys, non-zero term frequencies — the C side of the boundary refuses what the reference's types cannot hold."""
    m.check_vectors([0, 3, 3, 5], [1, 5, 9, 2, 7], [1, 2, 3, 1, 1])            # valid, incl. an empty vector
    m.check_vectors([0, 2], [4, 8])                                              # Query-like: no tfs
    for off, terms, tfs, what in [([0, 3], [1, 5, 5], [1, 1, 1], "strictly ascending"),      # duplicate key
                                  ([0, 3], [1, 9, 5], [1, 1, 1], "strictly ascending"),      # unsorted
                                  ([0, 2, 4], [1, 2, 3, 4], [1, 1, 0, 1], "zero term frequency"),
                                  ([0, 3, 2], [1, 2, 3], [1, 1, 1], "offsets not monotone"),
                                  ([0, 2], [7, 7], None, "strictly ascending")]:
        with pytest.raises(m.Bm25xError) as e:
            m.check_vectors(off, terms, tfs)
        assert e.value.code == 1 and "invalid data" in str(e.value) and what in str(e.value)
    # keys restart between vectors: each vector is checked on its own
    m.check_vectors([0, 2, 4], [5, 9, 1, 2], [1, 1, 1, 1])
