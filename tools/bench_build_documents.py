#!/usr/bin/env python
"""bench_build_documents.py — what building an index from documents costs on the GPU
(bm25x_index_create_from_documents) next to the host restatement of the reference's Segment plus bm25x_index_create.

Corpus: C3 of bench.py (its seeds: 10M documents, vocabulary 100k, 128 terms each), transposed to documents on the host
(doc-major, terms ascending inside each document), untimed.  Alternating the two arms round by round, the median of:
  gpu_ms    Index.from_documents end to end (host checks, df pass, inversion on the GPU; host clock around a call that ends
            in a synchronize)
  host_ms   the Segment on the host (a numpy stable sort of the mappings by term: they arrive in doc order, so the result
            is sorted by (term, doc); doc_len as the saturating Σ tf) plus Index() on that CSR
and, after the timed rounds, one more build under torch.profiler (CUDA activities) for the device time of each new kernel
and of the CUB sorts.  A keyed arm runs the same at `--keyed-docs` documents whose terms are random 16-byte keys (the
Segment's keys: a numpy sort of the keys as big-endian word pairs, then the same sort).  Both arms' handles must hold the same arrays (compared on the
device, slice by slice).  Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.

  python tools/bench_build_documents.py [--rounds 3] [--docs N] [--keyed-docs N]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_growing import card  # noqa: E402

KERNELS = ("k_df_count", "k_keys_be", "k_key_ordinals", "k_iota", "k_run_heads", "k_scatter", "DeviceRadixSort",
           "DeviceReduce")


def note(*a):
    print(*a, file=sys.stderr, flush=True)


def ms(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def transpose(m, c):
    """The documents of a term-major synthetic corpus: (elem_off u64, elem_term u32, elem_tf u32)."""
    import scipy.sparse
    mat = scipy.sparse.csc_matrix((c.post_tf, c.post_doc, c.post_off.astype(np.int64)), shape=(c.n_docs, c.n_terms))
    mat = mat.tocsr()
    term = mat.indices.view(np.uint32) if mat.indices.itemsize == 4 else mat.indices.astype(np.uint32)
    return mat.indptr.astype(np.uint64), term, mat.data


def host_segment(m, off, tf, term=None, key=None, n_terms=0):
    """The Segment of the documents (numpy) handed to Index()."""
    keys = None
    if key is not None:                                      # the distinct keys ascending bytewise, each element's rank
        w = np.ascontiguousarray(key).view(">u8").reshape(-1, 2)
        order = np.lexsort((w[:, 1], w[:, 0]))
        first = np.ones(len(order), bool)
        first[1:] = np.any(w[order[1:]] != w[order[:-1]], axis=1)
        term = np.empty(len(order), np.uint32)
        term[order] = np.cumsum(first) - 1
        keys = key[order[first]]
        n_terms = len(keys)
    n = len(off) - 1
    doc = np.repeat(np.arange(n, dtype=np.uint32), np.diff(off.astype(np.int64)))
    order = np.argsort(term, kind="stable")
    post_off = np.zeros(n_terms + 1, np.uint64)
    post_off[1:] = np.cumsum(np.bincount(term, minlength=n_terms))
    doc_len = np.minimum(np.bincount(doc, weights=tf, minlength=n), 0xFFFFFFFF).astype(np.uint32)
    return m.Index(n, doc_len, n_terms, post_off, doc[order], tf[order], term_keys=keys)


_rt = None


def _same_device(a, b, nbytes, piece=256 << 20):
    global _rt
    if _rt is None:
        _rt = ctypes.CDLL("libcudart.so.12") if os.path.exists("/usr/local/cuda/lib64/libcudart.so.12") else \
            ctypes.CDLL("libcudart.so")
        _rt.cudaMemcpy.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    x, y = np.empty(piece, np.uint8), np.empty(piece, np.uint8)
    for o in range(0, int(nbytes), piece):
        n = min(piece, int(nbytes) - o)
        assert _rt.cudaMemcpy(x.ctypes.data, a + o, n, 2) == 0 and _rt.cudaMemcpy(y.ctypes.data, b + o, n, 2) == 0
        if not np.array_equal(x[:n], y[:n]):
            return False
    return True


def same_handles(a, b):
    la, lb = a.layout(), b.layout()
    if any(getattr(la, f) != getattr(lb, f) for f in ("n_docs", "n_terms", "n_postings", "n_postings_padded", "n_blocks",
                                                       "sum_doc_len", "avgdl")):
        return False
    if any(la.bytes[i] != lb.bytes[i] or not _same_device(la.dev_ptr[i], lb.dev_ptr[i], lb.bytes[i]) for i in range(13)):
        return False
    da, db = a.derived(), b.derived()
    return all(getattr(da, f + "_bytes") == getattr(db, f + "_bytes") and
               _same_device(getattr(da, f), getattr(db, f), getattr(db, f + "_bytes")) for f in ("pdoc", "champ", "champ_off"))


def profiled(build):
    """Device time (ms) of each kernel family of one build from documents."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ix = build()
        torch.cuda.synchronize()
    ix.close()
    kern, h2d = {}, 0.0
    for ev in prof.events():
        name, dur = ev.name, ev.device_time_total / 1e3
        k = next((k for k in KERNELS if k in name), None)
        if k:
            kern[k] = kern.get(k, 0.0) + dur
        elif "Memcpy HtoD" in name or "Memcpy H2D" in name:
            h2d += dur
    return {k: round(v, 2) for k, v in kern.items()}, round(h2d, 1)


def arm_pair(m, rounds, docs, segment):
    """(gpu times, host times, handles equal, profile) of one corpus of documents."""
    build = lambda: m.Index.from_documents(**docs)
    build().close()                                          # warm-up: module load, first allocations
    t_gpu, t_host = [], []
    for _ in range(rounds):
        t, ix = ms(build)
        t_gpu.append(t)
        ix.close()
        t, ix = ms(segment)
        t_host.append(t)
        ix.close()
        note(f"round: gpu {t_gpu[-1]:.1f} ms, host {t_host[-1]:.1f} ms")
    a, b = build(), segment()
    equal = same_handles(a, b)
    a.close()
    b.close()
    kern, h2d = profiled(build)
    return {"gpu_ms": round(statistics.median(t_gpu), 1), "host_ms": round(statistics.median(t_host), 1),
            "gpu_ms_all": [round(x, 1) for x in t_gpu], "host_ms_all": [round(x, 1) for x in t_host],
            "device_kernel_ms": kern, "device_h2d_ms": h2d, "handles_equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--keyed-docs", type=int, default=1_000_000)
    a = ap.parse_args()
    import _pkg
    m = _pkg.load()
    m.load_library()
    seed, vocab = 0xB25C0DE0 + 3, 100_000
    out = {"bench": "build_documents", "rounds": a.rounds, "vocab": vocab, "card": card()}
    note(f"card: {out['card']}")

    c = m.synth_corpus(seed, a.docs, vocab, 128)
    off, term, tf = transpose(m, c)
    c.free()
    note(f"keyless: {a.docs} documents, {int(off[-1])} elements")
    out["keyless"] = {"docs": a.docs, "elements": int(off[-1]), **arm_pair(
        m, a.rounds, dict(elem_off=off, elem_tf=tf, elem_term=term, n_terms=vocab),
        lambda: host_segment(m, off, tf, term=term, n_terms=vocab))}
    del off, term, tf

    c = m.synth_corpus(seed, a.keyed_docs, vocab, 128)
    off, term, tf = transpose(m, c)
    c.free()
    keys = np.random.default_rng(seed).integers(0, 256, size=(vocab, 16), dtype=np.uint8)
    kw = keys.view(">u8").reshape(vocab, 2)
    rank = np.empty(vocab, np.int64)
    rank[np.lexsort((kw[:, 1], kw[:, 0]))] = np.arange(vocab)       # bytewise rank of each term's key
    doc = np.repeat(np.arange(a.keyed_docs), np.diff(off.astype(np.int64)))
    order = np.lexsort((rank[term], doc))                           # each document's elements ascending by key
    ek, etf = keys[term[order]], tf[order]
    del doc, order, term, tf
    note(f"keyed: {a.keyed_docs} documents, {int(off[-1])} elements")
    out["keyed"] = {"docs": a.keyed_docs, "elements": int(off[-1]), **arm_pair(
        m, a.rounds, dict(elem_off=off, elem_tf=etf, elem_key=ek), lambda: host_segment(m, off, etf, key=ek))}
    print(json.dumps(out))
    if not (out["keyless"]["handles_equal"] and out["keyed"]["handles_equal"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
