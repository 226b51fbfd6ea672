#!/usr/bin/env python
"""bench_evaluate_tsvectors.py — `<&>` from tsvectors on the GPU: bm25x_evaluate_tsvectors against the four-step route a
caller takes without it (the document cast downloaded with its keys, every key looked up on the host, the unknown keys
numbered past n_terms in key order and every row re-sorted by ordinal, the queries through bm25x_tsvector_queries, each
query repeated for its pairs, bm25x_evaluate_batch).

Index: `--index-docs` synthetic tsvectors (util_tsvector.synthetic: 40..120 distinct lexemes drawn Zipf-like from a
vocabulary of 100k words, 10% of them 16..64 bytes long).  Documents: `--docs` tsvectors of 80..120 lexemes from the
same words plus 10k unknown ones.  Two shapes:
  one_query   every document against one query of 8 lexemes (pair_query all 0), the common SQL shape
  own_query   every document against its own query of 1..8 lexemes (pair_query NULL)
Per shape: the one call's wall time (host clock around the call, which ends in a download), the median of `--rounds`;
the four-step route's wall time, one round (its host steps dominate); pairs/s of each; and, from one more call under
torch.profiler (CUDA activities), the device time of the casts' kernels (k_tsv_*, CUB's sort and reduce) and of
k_evaluate.  Both arms must give the same bits.  Prints one JSON line with the card's name and power limit, read in
the same run; writes nothing.

  python tools/bench_evaluate_tsvectors.py [--rounds 3] [--docs 200000] [--index-docs 100000]

The defaults are the size measured in DESIGN §4.2.  `--docs 1000000` (10^8 entries) is the 10^6-document shape; it has
not been measured.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_build_documents import ms, note  # noqa: E402
from bench_growing import card  # noqa: E402
from util_evaluate_tsvector import SEED, evaluate_pairs, four_step_pairs  # noqa: E402
from util_tsvector import pack_ids, synthetic, word_table  # noqa: E402


def profiled(call):
    """Device time (ms) of the casts' kernels and of k_evaluate in one call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    cast_ms = kernel_ms = h2d_ms = 0.0
    for ev in prof.events():
        name, dur = ev.name, ev.device_time_total / 1e3
        if "k_evaluate" in name:
            kernel_ms += dur
        elif "k_tsv_" in name or "cub" in name.lower():
            cast_ms += dur
        elif "Memcpy HtoD" in name or "Memcpy H2D" in name:
            h2d_ms += dur
    return round(cast_ms, 2), round(kernel_ms, 2), round(h2d_ms, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--index-docs", type=int, default=100_000)
    a = ap.parse_args()
    import _pkg
    m = _pkg.load()
    m.load_library()
    if m.device_count() < 1:
        raise SystemExit("bench_evaluate_tsvectors: no CUDA device (there is no CPU fallback)")
    out = {"bench": "evaluate_tsvectors", "docs": a.docs, "rounds": a.rounds, "card": card()}
    note(f"card: {out['card']}")
    rng = np.random.default_rng(0xB25C0DE0 + 7)
    tsv, words, _ = synthetic(rng, a.index_docs, 40, 120, 100_000, 0.1)
    ix = m.Index.from_tsvectors(SEED, **tsv)
    del tsv
    unknown = [b"unknown-%d" % i for i in range(10_000)]
    flat, off = word_table(words + unknown)
    V = len(words)
    p = np.concatenate([1.0 / np.arange(1, V + 1) ** 0.8 * 0.95 / (1.0 / np.arange(1, V + 1) ** 0.8).sum(),
                        np.full(len(unknown), 0.05 / len(unknown))])
    lens = rng.integers(80, 121, a.docs)
    wid = rng.choice(len(p), size=int(lens.sum()), p=p)
    docs = pack_ids(lens, flat, off, wid, rng.integers(1, 5, len(wid)))
    del wid
    out["doc_entries"] = int(docs["ent_off"][-1])
    note(f"{a.docs} document tsvectors, {out['doc_entries']} entries, {len(docs['data'])} area bytes")
    one = pack_ids([8], flat, off, rng.choice(2000, 8, replace=False), np.full(8, -1))
    qlens = rng.integers(1, 9, a.docs)
    qwid = rng.choice(len(p), size=int(qlens.sum()), p=p)
    own = pack_ids(qlens, flat, off, qwid, np.full(len(qwid), -1))
    del qwid
    shapes = {"one_query": (one, np.zeros(a.docs, np.uint32)), "own_query": (own, None)}
    for name, (queries, pq) in shapes.items():
        call = lambda: ix.evaluate_tsvectors(SEED, docs, queries, pq)
        call()                                                   # warm-up: tables, vocabulary copy, module load
        t_one = []
        for _ in range(a.rounds):
            t, got = ms(call)
            t_one.append(t)

        def route():
            pairs = four_step_pairs(m, ix, docs, queries, pq)
            rc, r = evaluate_pairs(m, ix.h, pairs)
            assert rc == 0, m.load_library().bm25x_last_error()
            return r[:a.docs]

        t_four, want = ms(route)
        same = bool(np.array_equal(got, want))
        cast_ms, kernel_ms, h2d_ms = profiled(call)
        one_ms = statistics.median(t_one)
        out[name] = {"one_call_ms": round(one_ms, 1), "one_call_pairs_per_s": round(a.docs / one_ms * 1e3),
                     "four_step_ms": round(t_four, 1), "four_step_pairs_per_s": round(a.docs / t_four * 1e3),
                     "speedup": round(t_four / one_ms, 2), "cast_kernels_ms": cast_ms, "k_evaluate_ms": kernel_ms,
                     "h2d_ms": h2d_ms, "same_bits": same, "nonzero": int(np.count_nonzero(got))}
        note(f"{name}: {out[name]}")
        if not same:
            print(json.dumps(out))
            raise SystemExit(f"{name}: the one call and the four-step route differ")
    ix.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
