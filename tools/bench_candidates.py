#!/usr/bin/env python
"""bench_candidates.py — per-query candidate lists (bm25x_search_candidates) against what the batch ABI offered before.

Workload: C3 of bench.py (its seeds: 10M documents, vocabulary 100k, 128 terms each) and its 100k 3-term top-10 queries,
each with its own candidate list of |C| documents, |C| in --sizes: half drawn from the documents holding one of the
query's terms, half uniformly (duplicates allowed, unsorted) — the shape a filter or an ANN pre-selection hands over.
Three arms, alternated round by round, median over the rounds:
  candidates   Index.search_candidates of all queries, one call
  batch        Index.search_batch of the same queries without a filter (the batched reference point; once per round)
  bitmap       Index.search_batch of one query with allow = the bitmap of its candidates, the way a per-query filter had
               to be sent before; timed per query on the first --subset queries
For each: end to end (host clock around the call, which ends in a synchronise) and device time (the call's stats.kernel_ms:
CUDA events around its kernels on the library's stream).  The rows of the candidate search must equal the bitmap
searches' on the subset, else the exit status is 1.  Prints one JSON line with the card's name and power limit, read in
the same run; writes nothing.

  python tools/bench_candidates.py [--rounds 3] [--docs N] [--queries Q] [--sizes 16,128,1024,8192] [--subset 300]
"""
import argparse
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

ROWS = ("doc", "score", "score64", "n")


def draw(rng, c, q_off, q_terms, size, chunk=8192):
    """(c_off, c_docs): per query `size` candidates, half from the holders of its terms, half uniform."""
    nq = len(q_off) - 1
    half = size // 2
    c_off = (np.arange(nq + 1, dtype=np.uint64) * size).astype(np.uint32)
    c_docs = np.empty(nq * size, np.uint32)
    df = np.diff(c.post_off.astype(np.int64))
    for a in range(0, nq, chunk):
        b = min(nq, a + chunk)
        n = b - a
        pick = rng.integers(0, 3, (n, half)) + q_off[a:b, None].astype(np.int64)   # one of the 3 terms
        t = q_terms[pick]
        pos = c.post_off[t].astype(np.int64) + (rng.random((n, half)) * df[t]).astype(np.int64)
        held = c.post_doc[pos]
        uni = rng.integers(0, c.n_docs, (n, size - half), dtype=np.uint32)
        block = np.concatenate([held, uni], axis=1)
        block = np.take_along_axis(block, rng.permuted(np.tile(np.arange(size), (n, 1)), axis=1), axis=1)
        c_docs[a * size:b * size] = block.ravel()
    return c_off, c_docs


def bitmap(docs, n):
    b = np.zeros((n + 7) // 8, np.uint8)
    d = np.asarray(docs, np.int64)
    np.bitwise_or.at(b, d >> 3, (1 << (d & 7)).astype(np.uint8))
    return b


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--sizes", default="16,128,1024,8192")
    ap.add_argument("--subset", type=int, default=300)
    a = ap.parse_args()
    import _pkg
    m = _pkg.load()
    m.load_library()
    seed, vocab, k = 0xB25C0DE0 + 3, 100_000, 10
    c = m.synth_corpus(seed, a.docs, vocab, 128)
    ix = m.Index.from_corpus(c)
    q_off, q_terms = m.synth_queries(seed + 1000, a.queries, vocab, 3, 3, c.post_off)
    assert np.all(np.diff(q_off) == 3)
    rng = np.random.default_rng(seed)
    sizes = [int(s) for s in a.sizes.split(",")]
    S = min(a.subset, a.queries)
    ix.search_batch(q_off, q_terms, k)                 # warm-up: module load, first allocations
    batch_e2e, batch_dev = [], []
    res = {}
    ok = True
    for size in sizes:
        c_off, c_docs = draw(rng, c, q_off, q_terms, size)
        bms = [bitmap(c_docs[c_off[i]:c_off[i + 1]], c.n_docs) for i in range(S)]
        ix.search_candidates(q_off, q_terms, c_off, c_docs, k)           # warm-up of this size
        r = {"cand_e2e": [], "cand_dev": [], "bitmap_e2e": [], "bitmap_dev": []}
        got = None
        for _ in range(a.rounds):
            t, got = timed(lambda: ix.search_candidates(q_off, q_terms, c_off, c_docs, k))
            r["cand_e2e"].append(t)
            r["cand_dev"].append(got["stats"].kernel_ms)
            t, b = timed(lambda: ix.search_batch(q_off, q_terms, k))
            batch_e2e.append(t)
            batch_dev.append(b["stats"].kernel_ms)
            e2e = dev = 0.0
            rows = []
            for i in range(S):
                t, one = timed(lambda: ix.search_batch(q_off[i:i + 2] - q_off[i], q_terms[q_off[i]:q_off[i + 1]], k,
                                                        allow=bms[i]))
                e2e += t
                dev += one["stats"].kernel_ms
                rows.append(one)
            r["bitmap_e2e"].append(e2e / S)
            r["bitmap_dev"].append(dev / S)
        equal = all(np.array_equal(got[key][i], rows[i][key][0]) for i in range(S) for key in ROWS)
        ok &= equal
        st = got["stats"]
        res[size] = {
            "candidates_ms": round(statistics.median(r["cand_e2e"]), 2),
            "candidates_device_ms": round(statistics.median(r["cand_dev"]), 3),
            "candidates_ms_all": [round(x, 2) for x in r["cand_e2e"]],
            "candidates_h2d_ms": round(st.h2d_ms, 2), "candidates_d2h_ms": round(st.d2h_ms, 2),
            "lookup_reads": int(st.postings_fetched),
            "bitmap_per_query_ms": round(statistics.median(r["bitmap_e2e"]), 3),
            "bitmap_per_query_device_ms": round(statistics.median(r["bitmap_dev"]), 4),
            "rows_equal_bitmap_search": bool(equal)}
        del c_off, c_docs, bms, got
    print(json.dumps({
        "bench": "candidates", "docs": a.docs, "queries": a.queries, "k": k, "rounds": a.rounds, "subset": S,
        "batch_unfiltered_ms": round(statistics.median(batch_e2e), 2),
        "batch_unfiltered_device_ms": round(statistics.median(batch_dev), 3),
        "sizes": res, "card": card()}))
    ix.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
