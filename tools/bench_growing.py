#!/usr/bin/env python
"""bench_growing.py — what the mutable growing segment costs next to re-creating an immutable growing handle.

Sealed: the C3 corpus of bench.py (its seeds: 10M documents, vocabulary 100k, 128 terms each) and its 100k 3-term top-10
queries.  Growing: `--growing` documents of the same vocabulary (another seed), inserted into a segment in batches of 1,
100 and 10 000 documents, the batch sizes alternating round by round.  Per batch size, the median over the rounds of:
  insert_ms          one bm25x_growing_insert call (through the Python binding), median over the round's calls
  refresh_fill_ms    bm25x_growing_refresh after all documents were inserted (every posting pending)
  refresh_batch_ms   bm25x_growing_refresh after one more batch of that size (the steady-state refresh)
  search_ms          the queries end to end through bm25x_growing_search_batch (nothing pending)
  create_ms          bm25x_growing_create over the same documents (what a re-created handle costs)
  search_create_ms   the queries end to end through bm25x_search_batch_growing on that handle
Both searches must return identical rows.  Prints one JSON line with the card's name and power limit; writes nothing.

  python tools/bench_growing.py [--rounds 3] [--steps 3] [--docs N] [--growing G] [--queries Q]
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
BATCHES = (1, 100, 10_000)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,power.max_limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit, max_limit = [x.strip() for x in out.split(",")[:3]]
        return {"name": name, "power_limit": limit, "power_max_limit": max_limit}
    except Exception as e:  # noqa: BLE001 — reported in the output
        return {"error": str(e)}


def doc_major(c):
    """The documents of a term-major synthetic corpus: (elem_off, elem_term, elem_tf, doc_len)."""
    df = np.diff(c.post_off.astype(np.int64))
    term = np.repeat(np.arange(c.n_terms, dtype=np.uint32), df)
    order = np.lexsort((term, c.post_doc))
    off = np.zeros(c.n_docs + 1, np.uint64)
    off[1:] = np.cumsum(np.bincount(c.post_doc, minlength=c.n_docs))
    return off, term[order], np.ascontiguousarray(c.post_tf[order]), np.array(c.doc_len, np.uint32)


def ms(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--growing", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=100_000)
    a = ap.parse_args()

    import _pkg
    m = _pkg.load()
    m.load_library()
    seed, vocab, k = 0xB25C0DE0 + 3, 100_000, 10                     # bench.py WORKLOADS["c3"]
    c = m.synth_corpus(seed, a.docs, vocab, 128, 128, 0.0)
    q_off, q_terms = m.synth_queries(seed + 1000, a.queries, vocab, 3, 3, c.post_off)
    ix = m.Index.from_corpus(c)
    c.free()
    gc = m.synth_corpus(seed + 77, a.growing, vocab, 128, 128, 0.0)
    off, term, tf, dlen = doc_major(gc)
    gc.free()
    G = len(dlen)

    def docs(lo, hi):
        return dict(elem_off=off[lo:hi + 1] - off[lo], elem_term=term[off[lo]:off[hi]], elem_tf=tf[off[lo]:off[hi]],
                    doc_len=dlen[lo:hi])

    res = {B: {x: [] for x in ("insert_ms", "refresh_fill_ms", "refresh_batch_ms", "search_ms", "create_ms",
                               "search_create_ms")} for B in BATCHES}
    identical = True
    for _ in range(a.rounds):
        for B in BATCHES:
            r = res[B]
            seg = ix.growing_segment()
            calls = [ms(lambda lo=lo: seg.insert(**docs(lo, min(lo + B, G - B))))[0] for lo in range(0, G - B, B)]
            r["insert_ms"].append(statistics.median(calls))
            r["refresh_fill_ms"].append(ms(seg.refresh)[0])
            seg.insert(**docs(G - B, G))
            r["refresh_batch_ms"].append(ms(seg.refresh)[0])
            seg.search_batch(q_off, q_terms, k)                            # warm-up
            r["search_ms"].append(statistics.median(ms(lambda: seg.search_batch(q_off, q_terms, k))[0]
                                                    for _ in range(a.steps)))
            got = seg.search_batch(q_off, q_terms, k, want_payload=True)
            seg.close()
            t, gh = ms(lambda: ix.growing(**docs(0, G)))
            r["create_ms"].append(t)
            ix.search_batch_growing(gh, q_off, q_terms, k)
            r["search_create_ms"].append(statistics.median(ms(lambda: ix.search_batch_growing(gh, q_off, q_terms, k))[0]
                                                           for _ in range(a.steps)))
            want = ix.search_batch_growing(gh, q_off, q_terms, k, want_payload=True)
            gh.close()
            identical &= all(np.array_equal(got[x], want[x]) for x in ("doc", "score", "score64", "payload", "n"))
    out = {"card": card(), "sealed_docs": a.docs, "growing_docs": G, "queries": a.queries, "k": k, "rounds": a.rounds,
           "rows_identical": bool(identical),
           "per_batch": {str(B): {x: round(statistics.median(v), 3) for x, v in res[B].items()} for B in BATCHES}}
    print(json.dumps(out))
    ix.close()
    return 0 if identical else 1


if __name__ == "__main__":
    sys.exit(main())
