#!/usr/bin/env python
"""bench_rebind.py — what the rebind of a growing segment to its seal's result (bm25x_growing_rebind) costs next to what a
caller had to do without it: open a fresh segment on the new index, insert the carried documents again, refresh.

Sealed: the C3 corpus of bench.py (its seeds: `--docs` documents, vocabulary 100k, 128 terms each).  Growing: `--growing`
documents of the same vocabulary (another seed), inserted in batches of 10 000, 1 % of them deleted, then sealed; then
`--carried` more documents (another seed) inserted after the seal's snapshot.  Each round builds that state afresh
(untimed) and times both arms on it, alternating their order round by round.  Each figure is taken twice: the host
clock around the call (which ends in a device synchronize) and device events recorded on the legacy default stream
before and after it (`*_ev_ms`).  The median of:
  seal_ms       bm25x_growing_seal of the growing documents
  rebind_ms     bm25x_growing_rebind of the segment to the seal's result
  reinsert_ms   the workaround: bm25x_growing_open on the new index, bm25x_growing_insert of the carried documents,
                bm25x_growing_refresh (the three calls)
Both segments must answer `--queries` 3-term top-10 queries with identical rows (payloads given, so that the carried
documents keep theirs in both).  Prints one JSON line with the card's name and power limit, read in the same run;
writes nothing.

  python tools/bench_rebind.py [--rounds 3] [--docs N] [--growing G] [--carried C] [--queries Q]
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

from bench_growing import card, doc_major  # noqa: E402


_rt = None


def ms(f):
    """(host ms, device-event ms, f()) of a call that ends in a device synchronize."""
    global _rt
    if _rt is None:
        _rt = ctypes.CDLL("libcudart.so.12") if os.path.exists("/usr/local/cuda/lib64/libcudart.so.12") else \
            ctypes.CDLL("libcudart.so")
        _rt.cudaEventRecord.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        _rt.cudaEventSynchronize.argtypes = [ctypes.c_void_p]
        _rt.cudaEventElapsedTime.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_void_p, ctypes.c_void_p]
        _rt.cudaEventDestroy.argtypes = [ctypes.c_void_p]
    ev = [ctypes.c_void_p(), ctypes.c_void_p()]
    for e in ev:
        assert _rt.cudaEventCreate(ctypes.byref(e)) == 0
    assert _rt.cudaEventRecord(ev[0], None) == 0
    t0 = time.perf_counter()
    r = f()
    host = (time.perf_counter() - t0) * 1e3
    assert _rt.cudaEventRecord(ev[1], None) == 0 and _rt.cudaEventSynchronize(ev[1]) == 0
    dev = ctypes.c_float()
    assert _rt.cudaEventElapsedTime(ctypes.byref(dev), ev[0], ev[1]) == 0
    for e in ev:
        _rt.cudaEventDestroy(e)
    return host, float(dev.value), r


def batches(seg, e_off, e_term, e_tf, dlen, pay):
    for lo in range(0, len(dlen), 10_000):
        hi = min(lo + 10_000, len(dlen))
        seg.insert(elem_off=e_off[lo:hi + 1] - e_off[lo], elem_term=e_term[e_off[lo]:e_off[hi]],
                   elem_tf=e_tf[e_off[lo]:e_off[hi]], doc_len=dlen[lo:hi], payload=pay[lo:hi])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--growing", type=int, default=1_000_000)
    ap.add_argument("--carried", type=int, default=50_000)
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
    c.free()
    docs = []
    for s, n in ((seed + 77, a.growing), (seed + 78, a.carried)):
        gc = m.synth_corpus(s, n, vocab, 128, 128, 0.0)
        docs.append(doc_major(gc) + (rng.integers(0, 65536, size=(n, 3)).astype(np.uint16),))
        gc.free()
    gdel = np.flatnonzero(rng.random(a.growing) < 0.01)

    res = {f"{x}{y}": [] for x in ("seal", "rebind", "reinsert") for y in ("_ms", "_ev_ms")}
    identical = True
    for r in range(a.rounds):
        seg = ix.growing_segment()
        batches(seg, *docs[0])
        seg.delete(gdel)
        seg.refresh()
        t, te, (nix, *_) = ms(lambda: seg.seal())
        res["seal_ms"].append(t)
        res["seal_ev_ms"].append(te)
        batches(seg, *docs[1])
        seg.refresh()
        ref = None
        for arm in (("rebind", "reinsert") if r % 2 == 0 else ("reinsert", "rebind")):
            if arm == "rebind":
                t, te, _ = ms(lambda: seg.rebind(nix))
            else:
                def reinsert():
                    s = nix.growing_segment()
                    batches(s, *docs[1])
                    s.refresh()
                    return s
                t, te, ref = ms(reinsert)
            res[arm + "_ms"].append(t)
            res[arm + "_ev_ms"].append(te)
        got, want = (s.search_batch(q_off, q_terms, k, want_payload=True) for s in (seg, ref))
        identical &= all(np.array_equal(got[x], want[x]) for x in ("doc", "score", "score64", "payload", "n"))
        info = seg.info()
        ref.close()
        seg.close()
        nix.close()
    out = {"card": card(), "sealed_docs": a.docs, "growing_docs": a.growing, "growing_deleted": int(len(gdel)),
           "carried_docs": a.carried, "carried_postings": int(info.n_postings), "queries": a.queries, "k": k,
           "rounds": a.rounds, "rows_identical": bool(identical),
           **{x: round(statistics.median(v), 1) for x, v in res.items()},
           "all": {x: [round(y, 1) for y in v] for x, v in res.items()}}
    print(json.dumps(out))
    ix.close()
    return 0 if identical else 1


if __name__ == "__main__":
    sys.exit(main())
