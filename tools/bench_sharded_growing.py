#!/usr/bin/env python
"""bench_sharded_growing.py — what a growing segment over a document-sharded index costs on one GPU, next to the
sharded search alone and to the growing segment over the unsharded index, and what its seal costs next to the unsharded
seal and to bm25x_sharded_create over the restated corpus.

Sealed: the C3 corpus of bench.py (its seeds: 10M documents, vocabulary 100k, 128 terms each), unsharded and sharded
S = 2 and S = 4 (default bounds, every shard on device 0), 1 % of its documents deleted at the seal.  Growing: 100 k
documents of 128 terms of the same vocabulary (another seed), inserted in batches of 10 000 into both segments, 1 % of
them deleted.  Per S, alternating the arms round by round, the median of:
  search_sharded_growing_ms  `--queries` 3-term top-10 queries end to end, bm25x_growing_search_batch on the sharded segment
  search_sharded_ms          the same queries, bm25x_sharded_search_batch alone (no growing documents)
  search_unsharded_growing_ms  the same queries, bm25x_growing_search_batch on the unsharded segment
  seal_sharded_ms            bm25x_growing_seal_sharded (host clock; the call ends in a device synchronize)
  seal_unsharded_ms          bm25x_growing_seal on the unsharded segment
  create_sharded_ms          bm25x_sharded_create over the restated corpus with the seal's bounds (restatement not timed)
The two growing searches must give identical rows, and so must the three sealed results; the seal's maps must equal the
restatement's.  Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.

  python tools/bench_sharded_growing.py [--rounds 3] [--docs N] [--growing G] [--queries Q]
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

from bench_growing import card, doc_major  # noqa: E402
from bench_seal import ctid, restated  # noqa: E402

ROWS = ("doc", "score", "score64", "payload", "n")


def ms(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def note(*x):
    print(*x, file=sys.stderr, flush=True)


def same(a, b):
    return all(np.array_equal(a[x], b[x]) for x in ROWS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--growing", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--shards", type=int, nargs="+", default=[2, 4])
    a = ap.parse_args()

    import _pkg
    m = _pkg.load()
    m.load_library()
    if m.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    seed, vocab, k = 0xB25C0DE0 + 3, 100_000, 10                     # bench.py WORKLOADS["c3"]
    rng = np.random.default_rng(5)
    c = m.synth_corpus(seed, a.docs, vocab, 128, 128, 0.0)
    q_off, q_terms = m.synth_queries(seed + 1000, a.queries, vocab, 3, 3, c.post_off)
    ix = m.Index.from_corpus(c)
    sdel = rng.random(a.docs) < 0.01
    packed = np.packbits(sdel.astype(np.uint8), bitorder="little")
    gc = m.synth_corpus(seed + 77, a.growing, vocab, 128, 128, 0.0)
    g_off, g_doc, g_tf = gc.post_off.copy(), gc.post_doc.copy(), gc.post_tf.copy()
    e_off, e_term, e_tf, dlen = doc_major(gc)
    gc.free()
    G = len(dlen)
    gdel = rng.random(G) < 0.01

    def fill(seg):
        for lo in range(0, G, 10_000):
            hi = min(lo + 10_000, G)
            seg.insert(elem_off=e_off[lo:hi + 1] - e_off[lo], elem_term=e_term[e_off[lo]:e_off[hi]],
                       elem_tf=e_tf[e_off[lo]:e_off[hi]], doc_len=dlen[lo:hi])
        seg.delete(np.flatnonzero(gdel))
        seg.refresh()

    seg = ix.growing_segment()
    fill(seg)
    note("built C3 and the unsharded segment")
    # the restated corpus, on the host, before any timing
    off, doc, tf, cnt, smap, gmap = restated(c, sdel, g_off, g_doc, g_tf, gdel)
    doc_len = np.concatenate([cnt[~sdel], dlen[~gdel]]).astype(np.uint32)
    payload = np.concatenate([ctid(np.flatnonzero(~sdel)), ctid(np.flatnonzero(~gdel))])
    n_docs = len(doc_len)
    note("restated the corpus")

    per_s = {}
    identical = maps_identical = True
    for S in a.shards:
        sx = m.ShardedIndex.from_corpus(c, n_shards=S)
        bounds = sx.doc_bounds()
        kept = [int((~sdel[bounds[s]:bounds[s + 1]]).sum()) for s in range(S)]
        kept[-1] += int((~gdel).sum())
        new_bounds = np.concatenate([[0], np.cumsum(kept)]).astype(np.uint32)
        sseg = sx.growing_segment()
        fill(sseg)
        res = {x: [] for x in ("search_sharded_growing_ms", "search_sharded_ms", "search_unsharded_growing_ms",
                               "seal_sharded_ms", "seal_unsharded_ms", "create_sharded_ms")}
        search_arms = {"search_sharded_growing_ms": lambda: sseg.search_batch(q_off, q_terms, k, want_payload=True),
                       "search_sharded_ms": lambda: sx.search_batch(q_off, q_terms, k, want_payload=True),
                       "search_unsharded_growing_ms": lambda: seg.search_batch(q_off, q_terms, k, want_payload=True)}
        for f in search_arms.values():   # warm every shape
            f()
        seal_arms = {"seal_sharded_ms": lambda: sseg.seal(sealed_deleted=packed),
                     "seal_unsharded_ms": lambda: seg.seal(sealed_deleted=packed),
                     "create_sharded_ms": lambda: (m.ShardedIndex(n_docs, doc_len, vocab, off, doc, tf, payload=payload,
                                                                  n_shards=len(new_bounds) - 1, doc_bounds=new_bounds),)}
        note(f"S={S}: built")
        for r in range(a.rounds):
            note(f"S={S}: round {r}")
            rows = {}
            for name in (list(search_arms) if r % 2 == 0 else list(search_arms)[::-1]):
                t, rows[name] = ms(search_arms[name])
                res[name].append(t)
            identical &= same(rows["search_sharded_growing_ms"], rows["search_unsharded_growing_ms"])
            sealed_rows = {}
            for name in (list(seal_arms) if r % 2 == 0 else list(seal_arms)[::-1]):
                t, out = ms(seal_arms[name])
                res[name].append(t)
                if name != "create_sharded_ms":
                    maps_identical &= bool(np.array_equal(out[1], smap) and np.array_equal(out[2], gmap))
                if name == "seal_sharded_ms":
                    identical &= bool(np.array_equal(out[0].doc_bounds(), new_bounds))
                sealed_rows[name] = out[0].search_batch(q_off, q_terms, k, want_payload=True)
                out[0].close()
            identical &= same(sealed_rows["seal_sharded_ms"], sealed_rows["seal_unsharded_ms"])
            identical &= same(sealed_rows["seal_sharded_ms"], sealed_rows["create_sharded_ms"])
        per_s[f"S={S}"] = {**{x: round(statistics.median(v), 2) for x, v in res.items()},
                           "all": {x: [round(y, 2) for y in v] for x, v in res.items()}}
        sseg.close()
        sx.close()
    out = {"card": card(), "sealed_docs": a.docs, "sealed_deleted": int(sdel.sum()), "growing_docs": G,
           "growing_deleted": int(gdel.sum()), "new_docs": n_docs, "new_postings": int(off[-1]), "queries": a.queries,
           "k": k, "rounds": a.rounds, "rows_identical": bool(identical), "maps_identical": bool(maps_identical), **per_s}
    print(json.dumps(out))
    seg.close()
    ix.close()
    c.free()
    return 0 if identical and maps_identical else 1


if __name__ == "__main__":
    sys.exit(main())
