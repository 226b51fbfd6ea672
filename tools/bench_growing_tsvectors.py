#!/usr/bin/env python
"""bench_growing_tsvectors.py — what an insert of tsvectors into the growing segment costs on the GPU
(bm25x_growing_insert_tsvectors) against the host path it replaces.

Sealed side: synthetic tsvectors of C3's shape (tools/bench_tsvectors.py: 128 distinct lexemes per document, Zipf-like
over 100k words, `--long-frac` of them hashed), built with Index.from_tsvectors, untimed.  Growing: batches of 1, 100
and 10 000 tsvectors of the same shape, about 10 % of their lexemes words the sealed side lacks.  Two segments over the
sealed index take the same batches, the arms alternated batch by batch:
  gpu_ms    GrowingSegment.insert_tsvectors
  host_ms   the caller's restatement: bm25x_intern per lexeme, a numpy sort and merge per vector, bm25x_lookup_terms,
            a dict numbering the fresh keys, a re-sort by ordinal, then GrowingSegment.insert
Then both segments are sealed (the owned keys against new_keys given by the caller) and timed.  Both segments' arrays
and both seals' arrays must be equal.  Prints one JSON line with the card's name and power limit; writes nothing.

  python tools/bench_growing_tsvectors.py [--rounds 3] [--docs N] [--long-frac F]
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

from bench_build_documents import ms, note, same_handles  # noqa: E402
from bench_growing import card  # noqa: E402
from util_index import read_back  # noqa: E402
from util_tsvector import cast, pack_ids, synthetic, word_table  # noqa: E402

SEED = bytes(range(32))
MISSING = 0xFFFFFFFF


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=250_000)
    ap.add_argument("--long-frac", type=float, default=0.1)
    a = ap.parse_args()
    import _pkg
    m = _pkg.load()
    m.load_library()
    bm = __import__(m.__name__ + ".bm25x", fromlist=["x"])
    vocab = 100_000
    out = {"bench": "growing_tsvectors", "rounds": a.rounds, "docs": a.docs, "vocab": vocab, "long_frac": a.long_frac,
           "card": card()}
    note(f"card: {out['card']}")
    rng = np.random.default_rng(0xB25C0DE0 + 5)
    tsv, words, _ = synthetic(rng, a.docs, 128, 128, vocab, a.long_frac)
    sealed = m.Index.from_tsvectors(SEED, **tsv)
    del tsv
    fresh = [b"fresh-%d-" % i + w for i, w in enumerate(words[:20_000])]
    pool = words + fresh
    flat, woff = word_table(pool)
    p = 1.0 / np.arange(1, len(words) + 1) ** 0.8
    p /= p.sum()

    def batch(n):
        wid = rng.choice(len(words), size=128 * n, p=p)
        new = rng.random(len(wid)) < 0.1
        wid[new] = len(words) + rng.integers(0, len(fresh), int(new.sum()))
        vec = np.repeat(np.arange(n), 128)
        pair = np.unique(vec.astype(np.int64) * len(pool) + wid)
        vec, wid = pair // len(pool), pair % len(pool)
        return pack_ids(np.bincount(vec, minlength=n), flat, woff, wid, rng.integers(1, 5, len(wid)))

    T = sealed.n_terms
    seg_gpu, seg_host = sealed.growing_segment(), sealed.growing_segment()
    numbered = {}

    def host_insert(t):
        lex = t["data"]
        e = t["entries"].astype(np.int64)
        start = np.repeat(t["byte_off"][:-1].astype(np.int64), np.diff(t["ent_off"].astype(np.int64))) + (e >> 12)
        ln = (e >> 1) & 0x7FF
        k = np.array([np.frombuffer(bm.intern(SEED, bytes(lex[s:s + n])), np.uint8) for s, n in zip(start, ln)])
        off, keys, tf = cast(bm.intern, SEED, t, keys=k.reshape(-1, 16))
        ords = sealed.lookup_terms(keys)
        miss = np.nonzero(ords == MISSING)[0]
        new = sorted({bytes(keys[i]) for i in miss} - set(numbered))
        base = T + len(numbered)
        numbered.update({key: base + r for r, key in enumerate(new)})
        for i in miss:
            ords[i] = numbered[bytes(keys[i])]
        n = len(off) - 1
        vec = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
        order = np.lexsort((ords, vec))
        lens = np.minimum(np.bincount(vec, weights=tf.astype(np.float64), minlength=n), 0xFFFFFFFF).astype(np.uint32)
        seg_host.insert(off, ords[order], tf[order], doc_len=lens)

    warm = batch(1)
    seg_gpu.insert_tsvectors(SEED, **warm)                              # warm-up: the vocabulary goes up once
    host_insert(warm)
    out["batches"] = {}
    for n in (1, 100, 10_000):
        t_gpu, t_host = [], []
        for _ in range(a.rounds):
            t = batch(n)
            tg, _ = ms(lambda: seg_gpu.insert_tsvectors(SEED, **t))
            th, _ = ms(lambda: host_insert(t))
            t_gpu.append(tg)
            t_host.append(th)
        out["batches"][str(n)] = {"gpu_ms": round(statistics.median(t_gpu), 2), "host_ms": round(statistics.median(t_host), 2),
                                  "gpu_ms_all": [round(x, 2) for x in t_gpu], "host_ms_all": [round(x, 2) for x in t_host]}
        note(f"batch {n}: {out['batches'][str(n)]}")
    seg_gpu.refresh()
    seg_host.refresh()
    ga, gb = read_back(*seg_gpu.arrays()), read_back(*seg_host.arrays())
    keys = np.zeros((len(numbered), 16), np.uint8)
    for key, t in numbered.items():
        keys[t - T] = np.frombuffer(key, np.uint8)
    out["new_keys"] = len(numbered)
    out["segments_equal"] = bool(all(ga[x].tobytes() == gb[x].tobytes() for x in ga) and
                                 np.array_equal(seg_gpu.new_keys(), keys))
    t_own, t_given = [], []
    for _ in range(3):
        t, r_own = ms(lambda: seg_gpu.seal())
        t_own.append(t)
        t, r_given = ms(lambda: seg_host.seal(new_keys=keys))
        t_given.append(t)
    out["seal_owned_keys_ms"] = round(statistics.median(t_own), 1)
    out["seal_given_keys_ms"] = round(statistics.median(t_given), 1)
    out["seals_equal"] = bool(same_handles(r_own[0], r_given[0]) and
                              all(np.array_equal(x, y) for x, y in zip(r_own[1:], r_given[1:])))
    print(json.dumps(out))
    if not (out["segments_equal"] and out["seals_equal"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
