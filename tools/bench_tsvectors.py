#!/usr/bin/env python
"""bench_tsvectors.py — what taking documents and queries as tsvectors costs on the GPU (bm25x_cast_tsvectors,
bm25x_index_create_from_tsvectors, bm25x_tsvector_queries).

Corpus: synthetic tsvectors of C3's shape (128 distinct lexemes per document drawn Zipf-like from a vocabulary of 100k
words, `--long-frac` of the words 16..64 bytes long (the BLAKE3 path), the rest 1..15 (the copy path), 1..4 positions
each), made in numpy from a seed, untimed.  Alternating the three arms round by round, the median of:
  cast_ms         bm25x_cast_tsvectors (document mode) alone, host clock: upload, intern, sort, merge, download
  tsvectors_ms    Index.from_tsvectors end to end
  documents_ms    Index.from_documents on the same keyed documents, computed beforehand (numpy restatement of the cast)
The handles of the last two must hold the same arrays (compared on the device).  Then a batch of `--queries` query
tsvectors (1..8 words, some unknown to the index): Index.tsvector_queries against the host path it replaces, one
bm25x_intern call per lexeme, a numpy sort + dedup per query and bm25x_lookup_terms; both must give the same rows.
Prints one JSON line with the card's name and power limit, read in the same run; writes nothing.

  python tools/bench_tsvectors.py [--rounds 3] [--docs N] [--long-frac F] [--queries N]
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
from util_tsvector import cast, pack, synthetic  # noqa: E402

SEED = bytes(range(32))


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
    out = {"bench": "tsvectors", "rounds": a.rounds, "docs": a.docs, "vocab": vocab, "long_frac": a.long_frac,
           "card": card()}
    note(f"card: {out['card']}")
    rng = np.random.default_rng(0xB25C0DE0 + 3)
    tsv, words, wid = synthetic(rng, a.docs, 128, 128, vocab, a.long_frac)
    E = len(tsv["entries"])
    in_bytes = 4 * E + len(tsv["data"]) + 16 * (a.docs + 1)
    wkeys = np.array([np.frombuffer(bm.intern(SEED, w), np.uint8) for w in words])
    off, keys, tf = cast(bm.intern, SEED, tsv, keys=wkeys[wid])
    note(f"{a.docs} tsvectors, {E} entries, {len(tsv['data'])} area bytes, {int(off[-1])} cast elements")
    out.update(entries=E, input_bytes=in_bytes, hashed_entries=int(sum(len(words[i]) >= 16 for i in np.unique(wid))))

    c = bm.cast_tsvectors(SEED, **tsv)                                 # warm-up, and the cast against its restatement
    out["cast_equal"] = bool(np.array_equal(c[0], off) and np.array_equal(c[1], keys) and np.array_equal(c[2], tf))
    del c
    m.Index.from_documents(off, tf, elem_key=keys).close()
    t_cast, t_tsv, t_doc = [], [], []
    for _ in range(a.rounds):
        t, r = ms(lambda: bm.cast_tsvectors(SEED, **tsv))
        t_cast.append(t)
        del r
        t, ix = ms(lambda: m.Index.from_tsvectors(SEED, **tsv))
        t_tsv.append(t)
        ix.close()
        t, ix = ms(lambda: m.Index.from_documents(off, tf, elem_key=keys))
        t_doc.append(t)
        ix.close()
        note(f"round: cast {t_cast[-1]:.1f} ms, from_tsvectors {t_tsv[-1]:.1f} ms, from_documents {t_doc[-1]:.1f} ms")
    ix, ixd = m.Index.from_tsvectors(SEED, **tsv), m.Index.from_documents(off, tf, elem_key=keys)
    med = statistics.median(t_cast)
    out.update(cast_ms=round(med, 1), cast_entries_per_s=round(E / med * 1e3), cast_bytes_per_s=round(in_bytes / med * 1e3),
               tsvectors_ms=round(statistics.median(t_tsv), 1), documents_ms=round(statistics.median(t_doc), 1),
               cast_ms_all=[round(x, 1) for x in t_cast], tsvectors_ms_all=[round(x, 1) for x in t_tsv],
               documents_ms_all=[round(x, 1) for x in t_doc], handles_equal=bool(same_handles(ix, ixd)))
    ixd.close()

    # queries: 1..8 words, 1 in 8 of them unknown to the index
    nq = a.queries
    qlen = rng.integers(1, 9, nq)
    qw = [words[i] if rng.random() >= 0.125 else b"unknown-%d" % i for i in rng.integers(0, len(words), int(qlen.sum()))]
    qtsv = pack(qlen, qw, [1] * len(qw))
    ix.tsvector_queries(SEED, **qtsv)                                  # warm-up: the vocabulary goes to the device once

    def host():
        k = np.array([np.frombuffer(bm.intern(SEED, w), np.uint8) for w in qw]).reshape(-1, 16)
        qo, qk, _ = cast(bm.intern, SEED, qtsv, as_query=True, keys=k)
        return qo.astype(np.uint32), ix.lookup_terms(qk)

    t_gq, t_hq = [], []
    for _ in range(a.rounds):
        t, g = ms(lambda: ix.tsvector_queries(SEED, **qtsv))
        t_gq.append(t)
        t, h = ms(host)
        t_hq.append(t)
        note(f"queries: gpu {t_gq[-1]:.1f} ms, host {t_hq[-1]:.1f} ms")
    same = bool(np.array_equal(g[0], h[0]) and np.array_equal(g[1], h[1]))
    out["queries"] = {"n": nq, "lexemes": len(qw), "gpu_ms": round(statistics.median(t_gq), 1),
                      "host_ms": round(statistics.median(t_hq), 1), "gpu_ms_all": [round(x, 1) for x in t_gq],
                      "host_ms_all": [round(x, 1) for x in t_hq], "rows_equal": same}
    ix.close()
    print(json.dumps(out))
    if not (out["cast_equal"] and out["handles_equal"] and same):
        sys.exit(1)


if __name__ == "__main__":
    main()
