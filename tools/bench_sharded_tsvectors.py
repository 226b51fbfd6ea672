#!/usr/bin/env python
"""bench_sharded_tsvectors.py — what building a document-sharded index straight from tsvectors costs
(bm25x_index_create_sharded_from_tsvectors), against the unsharded build from tsvectors and the sharded build from the
documents of a cast made beforehand.

Corpus: synthetic tsvectors of C3's shape (128 distinct lexemes per document drawn Zipf-like from a vocabulary of 100k
words, `--long-frac` of the words 16..64 bytes long (the BLAKE3 path), the rest 1..15, 1..4 positions each), made in
numpy from a seed, untimed, with its document cast restated in numpy.  Alternating the arms round by round, the median
build wall time (host clock, end to end) of:
  unsharded_ms     Index.from_tsvectors
  tsvectors_S<s>   ShardedIndex.from_tsvectors, s shards, all on device 0
  documents_S<s>   ShardedIndex.from_documents on the precomputed cast, with the bounds the tsvector build chose
The sharded handles of both sources must hold the same arrays, shard for shard (compared on the device), and
`--queries` 3-term queries (from tsvectors, cast on the GPU) must give the same rows on every handle.  Peak device
memory of each build is sampled: the lowest free memory a polling thread sees while it runs, against the free memory
before it.  Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.

  python tools/bench_sharded_tsvectors.py [--rounds 3] [--docs N] [--long-frac F] [--queries N]
"""
import argparse
import json
import os
import statistics
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_build_documents import ms, note, same_handles  # noqa: E402
from bench_growing import card  # noqa: E402
from util_cuda import free_bytes  # noqa: E402
from util_tsvector import cast, pack, synthetic  # noqa: E402

SEED = bytes(range(32))
SHARDS = (2, 4)


class Shard:
    """Shard s of a sharded index as same_handles takes a handle."""

    def __init__(self, sx, s):
        self.lay, self.der = sx.shard_arrays(s)

    def layout(self):
        return self.lay

    def derived(self):
        return self.der


def same_sharded(a, b):
    bounds = a.doc_bounds()
    return bool(np.array_equal(bounds, b.doc_bounds()) and
                all(same_handles(Shard(a, s), Shard(b, s)) for s in range(len(bounds) - 1)))


def peak_bytes(build):
    """Device memory a build takes at its peak, sampled: free memory before it minus the lowest a polling thread sees."""
    before = free_bytes()
    low, done = [before], threading.Event()

    def poll():
        while not done.is_set():
            low[0] = min(low[0], free_bytes())

    t = threading.Thread(target=poll)
    t.start()
    try:
        h = build()
    finally:
        done.set()
        t.join()
    h.close()
    return before - low[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=250_000)
    ap.add_argument("--long-frac", type=float, default=0.1)
    ap.add_argument("--queries", type=int, default=100_000)
    a = ap.parse_args()
    import _pkg
    m = _pkg.load()
    m.load_library()
    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    vocab = 100_000
    out = {"bench": "sharded_tsvectors", "rounds": a.rounds, "docs": a.docs, "vocab": vocab, "long_frac": a.long_frac,
           "card": card()}
    note(f"card: {out['card']}")
    rng = np.random.default_rng(0xB25C0DE0 + 5)
    tsv, words, wid = synthetic(rng, a.docs, 128, 128, vocab, a.long_frac)
    E = len(tsv["entries"])
    wkeys = np.array([np.frombuffer(bm.intern(SEED, w), np.uint8) for w in words])
    off, keys, tf = cast(bm.intern, SEED, tsv, keys=wkeys[wid])
    note(f"{a.docs} tsvectors, {E} entries, {len(tsv['data'])} area bytes, {int(off[-1])} cast elements")
    out.update(entries=E, elements=int(off[-1]))

    arms = {"unsharded_ms": lambda: m.Index.from_tsvectors(SEED, **tsv)}
    bounds = {}
    for S in SHARDS:
        sx = m.ShardedIndex.from_tsvectors(SEED, **tsv, n_shards=S, devices=[0] * S)   # warm-up, and the bounds
        bounds[S] = sx.doc_bounds()
        sx.close()
        arms[f"tsvectors_S{S}_ms"] = lambda S=S: m.ShardedIndex.from_tsvectors(SEED, **tsv, n_shards=S, devices=[0] * S)
        arms[f"documents_S{S}_ms"] = lambda S=S: m.ShardedIndex.from_documents(off, tf, elem_key=keys, n_shards=S,
                                                                               doc_bounds=bounds[S], devices=[0] * S)
    m.Index.from_tsvectors(SEED, **tsv).close()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, build in arms.items():
            t, h = ms(build)
            times[name].append(t)
            h.close()
        note("round: " + ", ".join(f"{k} {v[-1]:.1f}" for k, v in times.items()))
    for k, v in times.items():
        out[k] = round(statistics.median(v), 1)
        out[k + "_all"] = [round(x, 1) for x in v]
    out["peak_device_bytes_sampled"] = {k[:-3]: peak_bytes(build) for k, build in arms.items()}
    out["bounds"] = {str(S): bounds[S].tolist() for S in SHARDS}

    ix = m.Index.from_tsvectors(SEED, **tsv)
    handles = {}
    equal = True
    for S in SHARDS:
        handles[f"tsvectors_S{S}"] = m.ShardedIndex.from_tsvectors(SEED, **tsv, n_shards=S, devices=[0] * S)
        handles[f"documents_S{S}"] = arms[f"documents_S{S}_ms"]()
        equal &= same_sharded(handles[f"tsvectors_S{S}"], handles[f"documents_S{S}"])
    out["handles_equal"] = equal

    # 3-term queries over the corpus' words, 1 in 8 words unknown to the index
    nq = a.queries
    qw = [words[i] if rng.random() >= 0.125 else b"unknown-%d" % i for i in rng.integers(0, len(words), 3 * nq)]
    qtsv = pack(np.full(nq, 3), qw, [1] * len(qw))
    q_off, q_terms = ix.tsvector_queries(SEED, **qtsv)
    want = ix.search_batch(q_off, q_terms, 10)
    rows = True
    for name, h in handles.items():
        qo, qt = h.tsvector_queries(SEED, **qtsv)
        rows &= bool(np.array_equal(qo, q_off) and np.array_equal(qt, q_terms))
        got = h.search_batch(qo, qt, 10)
        rows &= all(np.array_equal(got[k], want[k]) for k in ("doc", "score", "score64", "n"))
        h.close()
    ix.close()
    out["queries"] = {"n": nq, "k": 10, "rows_equal": rows}
    print(json.dumps(out))
    if not (equal and rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
