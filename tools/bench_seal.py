#!/usr/bin/env python
"""bench_seal.py — what the seal of a growing segment on the GPU (bm25x_growing_seal) costs next to what a caller can do
without it: restate the corpus on the host and upload it again with bm25x_index_create.

Sealed: the C3 corpus of bench.py (its seeds: 10M documents, vocabulary 100k, 128 terms each), 1 % of its documents
deleted.  Growing: `--growing` documents of the same vocabulary (another seed), inserted in batches of 10 000, 1 % of them
deleted.  The restated corpus (maintain.rs: sealed survivors relabelled, their length = their postings, then the growing
survivors) is built once on the host before the timing.  Alternating the two arms round by round, the median of:
  seal_ms      bm25x_growing_seal through the Python binding (host clock; the call ends in a device synchronize)
  create_ms    bm25x_index_create over the restated corpus from host memory (host clock, the same)
  roundtrip_ms the seal's per-document traffic over PCIe (lengths and payloads down, norms and payloads up), alone
Both results must answer `--queries` 3-term top-10 queries with identical rows (payloads included), and the seal's maps
must equal the restatement's.  Prints one JSON line with the card's name and power limit, read in the same run; writes
nothing.

  python tools/bench_seal.py [--rounds 3] [--docs N] [--growing G] [--queries Q]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_growing import card, doc_major  # noqa: E402


def ms(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def restated(c, sdel, g_off, g_doc, g_tf, gdel):
    """maintain.rs over a term-major sealed corpus c and a term-major growing CSR (doc ids = ordinals): per term the
    sealed survivors under their new ids, then the growing survivors after them; lengths = postings per sealed
    survivor (add_element), Σ tf per growing survivor."""
    N_s = c.n_docs
    smap = np.cumsum(~sdel, dtype=np.int64) - 1
    n_keep = int(smap[-1]) + 1
    gmap = n_keep + np.cumsum(~gdel, dtype=np.int64) - 1
    smap, gmap = smap.astype(np.uint32), gmap.astype(np.uint32)
    T = c.n_terms
    off = np.zeros(T + 1, np.uint64)
    cap = int(c.post_off[T]) + len(g_doc)
    doc, tf = np.empty(cap, np.uint32), np.empty(cap, np.uint32)
    keep_s, keep_g = ~sdel, ~gdel
    w = 0
    for t in range(T):
        o0, o1 = int(c.post_off[t]), int(c.post_off[t + 1])
        sd = c.post_doc[o0:o1]
        k = keep_s[sd]
        n = int(k.sum())
        doc[w:w + n] = smap[sd[k]]
        tf[w:w + n] = c.post_tf[o0:o1][k]
        w += n
        g0, g1 = int(g_off[t]), int(g_off[t + 1])
        gd = g_doc[g0:g1]
        k = keep_g[gd]
        n = int(k.sum())
        doc[w:w + n] = gmap[gd[k]]
        tf[w:w + n] = g_tf[g0:g1][k]
        w += n
        off[t + 1] = w
    cnt = np.bincount(c.post_doc, minlength=N_s)
    smap[sdel], gmap[gdel] = 0xFFFFFFFF, 0xFFFFFFFF   # the seal's maps: deleted documents have no new id
    return off, doc[:w], tf[:w], cnt, smap, gmap


def ctid(ids):
    """The synthetic payload of doc ids (a 291-tuple page), [n, 3] u16: what a document created without one keeps."""
    g = np.asarray(ids, np.int64)
    return np.stack([(g // 291) >> 16, (g // 291) & 0xFFFF, g % 291 + 1], axis=1).astype(np.uint16)


def roundtrip_ms(n_sealed, n_new, reps=5):
    """What the seal's per-document round trip costs alone: a D2H of 10 B per sealed document (lengths + payloads) and
    an H2D of 7 B per new document (fieldnorms + payloads), pageable host memory as the library uses; median ms."""
    import ctypes
    rt = ctypes.CDLL("libcudart.so")
    rt.cudaMalloc.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t]
    rt.cudaMemcpy.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    rt.cudaFree.argtypes = [ctypes.c_void_p]
    down, up = 10 * n_sealed, 7 * n_new
    dev = ctypes.c_void_p()
    assert rt.cudaMalloc(ctypes.byref(dev), max(down, up)) == 0
    host = np.empty(max(down, up), np.uint8)
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        assert rt.cudaMemcpy(host.ctypes.data, dev, down, 2) == 0
        assert rt.cudaMemcpy(dev, host.ctypes.data, up, 1) == 0
        out.append((time.perf_counter() - t0) * 1e3)
    rt.cudaFree(dev)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--growing", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=100_000)
    a = ap.parse_args()

    import _pkg
    m = _pkg.load()
    m.load_library()
    seed, vocab, k = 0xB25C0DE0 + 3, 100_000, 10                     # bench.py WORKLOADS["c3"]
    rng = np.random.default_rng(5)
    c = m.synth_corpus(seed, a.docs, vocab, 128, 128, 0.0)
    q_off, q_terms = m.synth_queries(seed + 1000, a.queries, vocab, 3, 3, c.post_off)
    ix = m.Index.from_corpus(c)
    sdel = rng.random(a.docs) < 0.01
    gc = m.synth_corpus(seed + 77, a.growing, vocab, 128, 128, 0.0)
    g_off, g_doc, g_tf = gc.post_off.copy(), gc.post_doc.copy(), gc.post_tf.copy()
    e_off, e_term, e_tf, dlen = doc_major(gc)
    gc.free()
    G = len(dlen)
    gdel = rng.random(G) < 0.01
    seg = ix.growing_segment()
    for lo in range(0, G, 10_000):
        hi = min(lo + 10_000, G)
        seg.insert(elem_off=e_off[lo:hi + 1] - e_off[lo], elem_term=e_term[e_off[lo]:e_off[hi]],
                   elem_tf=e_tf[e_off[lo]:e_off[hi]], doc_len=dlen[lo:hi])
    seg.delete(np.flatnonzero(gdel))
    seg.refresh()
    # the restated corpus, on the host
    off, doc, tf, cnt, smap, gmap = restated(c, sdel, g_off, g_doc, g_tf, gdel)
    c.free()
    doc_len = np.concatenate([cnt[~sdel], dlen[~gdel]]).astype(np.uint32)
    payload = np.concatenate([ctid(np.flatnonzero(~sdel)), ctid(np.flatnonzero(~gdel))])
    n_docs = len(doc_len)
    packed = np.packbits(sdel.astype(np.uint8), bitorder="little")

    res = {"seal_ms": [], "create_ms": []}
    identical = maps_identical = True
    for r in range(a.rounds):
        arms = ("seal", "create") if r % 2 == 0 else ("create", "seal")
        rows = {}
        for arm in arms:
            if arm == "seal":
                t, (nix, sm, gm, _) = ms(lambda: seg.seal(sealed_deleted=packed))
                maps_identical &= bool(np.array_equal(sm, smap) and np.array_equal(gm, gmap))
            else:
                t, nix = ms(lambda: m.Index(n_docs, doc_len, vocab, off, doc, tf, payload=payload))
            res[arm + "_ms"].append(t)
            rows[arm] = nix.search_batch(q_off, q_terms, k, want_payload=True)
            nix.close()
        identical &= all(np.array_equal(rows["seal"][x], rows["create"][x]) for x in ("doc", "score", "score64", "payload", "n"))
    out = {"card": card(), "sealed_docs": a.docs, "sealed_deleted": int(sdel.sum()), "growing_docs": G,
           "growing_deleted": int(gdel.sum()), "new_docs": n_docs, "new_postings": int(off[-1]), "queries": a.queries,
           "k": k, "rounds": a.rounds, "rows_identical": bool(identical), "maps_identical": bool(maps_identical),
           "roundtrip_ms": round(roundtrip_ms(a.docs, n_docs), 1),
           **{x: round(statistics.median(v), 1) for x, v in res.items()}, "all": {x: [round(y, 1) for y in v] for x, v in res.items()}}
    print(json.dumps(out))
    seg.close()
    ix.close()
    return 0 if identical and maps_identical else 1


if __name__ == "__main__":
    sys.exit(main())
