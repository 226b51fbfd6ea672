#!/usr/bin/env python
"""Where a seeded search warp's cycles go: builds the -DBM25X_PHASE_PROF variant of the library
(tools/build_variants.sh, variants/libbm25x_phaseprof.so), runs the C3 batch of bench.py on it and prints each phase's
share of the warp cycles of the seeded k <= 32 launches and its average per chunk.

  python tools/phase_profile.py [--docs N] [--queries N] [--runs R] [--no-build] [--json FILE]

The clock reads of the profile cost issue slots and order the code around them: the table attributes time, it is no
benchmark number (bench.py is).
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, "vectorchord-bm25_b200", "variants", "libbm25x_phaseprof.so")

# order of the PP_* enum in bm25x_search_ring.cuh
PHASES = ["query start / end", "refill wait", "window setup", "map clear", "seed listing", "stream trips",
          "compaction", "verify: ring searches", "flush: word-load wait", "hit append; flush: filter+exact+pool",
          "chunk end / refill issue"]
COUNTERS = ["chunks", "listed candidates", "hits", "flushes", "rows"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--no-build", action="store_true", help="use the variant library as it is")
    ap.add_argument("--json", help="also write the table as JSON to this file")
    a = ap.parse_args()
    if not a.no_build:
        subprocess.check_call(["bash", os.path.join(ROOT, "tools", "build_variants.sh"), "phaseprof=-DBM25X_PHASE_PROF"])
    os.environ["BM25X_LIBRARY"] = LIB  # read when the binding loads the library
    import _pkg
    m = _pkg.load()
    prof = ctypes.CDLL(LIB).bm25x_phase_prof
    prof.restype = ctypes.c_int
    prof.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    n = prof(None, 0)
    assert n == len(PHASES) + len(COUNTERS), n

    # the C3 batch of bench.py (same seeds)
    seed = 0xB25C0DE0 + 3
    c = m.synth_corpus(seed, a.docs, 100_000, 128, 128, 0.0)
    ix = m.Index.from_corpus(c)
    q_off, q_terms = m.synth_queries(seed + 1000, a.queries, 100_000, 3, 3, c.post_off, 0.0)
    b = ix.prepare(q_off, q_terms, a.k)
    b.run()  # warm-up
    prof(None, 1)
    ms = [b.run().kernel_ms for _ in range(a.runs)]
    buf = (ctypes.c_ulonglong * n)()
    prof(buf, 0)
    b.close()

    v = list(buf)
    cyc, cnt = v[:len(PHASES)], dict(zip(COUNTERS, v[len(PHASES):]))
    total = max(1, sum(cyc))
    chunks = max(1, cnt["chunks"])
    rows = [{"phase": ph, "share": c_ / total, "cycles_per_chunk": c_ / chunks} for ph, c_ in zip(PHASES, cyc)]
    print(f"seeded k<=32 launches, {a.runs} runs of {a.queries} queries on {a.docs} docs "
          f"(profiled kernel time {min(ms):.2f} ms: not a benchmark number)")
    print(f"{'phase':38s} {'share':>7s} {'cycles/chunk':>13s}")
    for r in rows:
        print(f"{r['phase']:38s} {100 * r['share']:6.1f}% {r['cycles_per_chunk']:13.0f}")
    print(f"{'total':38s} {100.0:6.1f}% {total / chunks:13.0f}")
    per_run = {k_: v_ / a.runs for k_, v_ in cnt.items()}
    print("per run: " + ", ".join(f"{k_} {v_:,.0f}" for k_, v_ in per_run.items()) +
          f"; per chunk: {cnt['listed candidates'] / chunks:.2f} listed, {cnt['hits'] / chunks:.2f} hits"
          f"; hit-list rows per flush: {cnt['rows'] / max(1, cnt['flushes']):.2f}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"rows": rows, "counters": cnt, "runs": a.runs, "kernel_ms": ms}, fh, indent=1)


if __name__ == "__main__":
    main()
