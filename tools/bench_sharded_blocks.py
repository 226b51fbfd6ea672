#!/usr/bin/env python
"""bench_sharded_blocks.py — what building a document-sharded index from the stored blocks costs, on the C3 corpus
(bench.py's corpus and query seeds), encoded in the reference's block codec by the oracle (oracle.oracle.EncodedBlocks).

Build wall time and device_bytes of:
  * the unsharded stored-block ingest (bm25x_index_create_from_blocks);
  * the sharded build from the blocks (bm25x_index_create_sharded_from_blocks) at S = 1, 2 and 4 on one GPU, and at
    S = 2 with one shard per device when two GPUs are visible;
  * the sharded build from the CSR (bm25x_sharded_create) at S = 4.
One arm is resident at a time (built, searched, closed); the arms alternate round by round.  In the first round every
arm answers bench.py's C3 queries and its rows must be identical to the unsharded ingest's.  Prints one JSON line; writes
nothing.

  python tools/bench_sharded_blocks.py [--rounds 3] [--docs N] [--queries Q] [--k 10]
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

from bench_sharded import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--k", type=int, default=10)
    a = ap.parse_args()
    import _pkg
    from oracle import oracle as orc
    orc.build()
    m = _pkg.load()
    m.load_library()
    seed, vocab, k, nq = 0xB25C0DE0 + 3, 100_000, a.k, a.queries      # bench.py WORKLOADS["c3"]
    t0 = time.time()
    c = m.synth_corpus(seed, a.docs, vocab, 128, 128, 0.0)
    q_off, q_terms = m.synth_queries(seed + 1000, nq, vocab, 3, 3, c.post_off)
    t_gen = time.time() - t0
    t0 = time.time()
    eb = orc.EncodedBlocks(orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf))
    t_enc = time.time() - t0
    blocks = dict(n_docs=c.n_docs, n_terms=c.n_terms, term_blk_off=eb.term_blk_off, blk_min_doc=eb.blk_min,
                  blk_n=eb.blk_n, blk_meta_doc=eb.meta_doc, blk_meta_tf=eb.meta_tf, blk_doc_off=eb.doc_off,
                  blk_tf_off=eb.tf_off, data=eb.bytes[:eb.n_bytes], doc_len=c.doc_len)

    arms = {"from_blocks unsharded": lambda: m.Index.from_blocks(**blocks)}
    for S in (1, 2, 4):
        arms[f"sharded_from_blocks S={S}"] = lambda S=S: m.ShardedIndex.from_blocks(**blocks, n_shards=S)
    if m.device_count() >= 2:
        arms["sharded_from_blocks S=2 on devices 0,1"] = lambda: m.ShardedIndex.from_blocks(**blocks, n_shards=2,
                                                                                            devices=[0, 1])
    arms["sharded_create S=4 (CSR)"] = lambda: m.ShardedIndex.from_corpus(c, n_shards=4)
    build_s = {name: [] for name in arms}
    device_bytes, identical, ref = {}, {}, None
    for rnd in range(a.rounds):
        for name, build in arms.items():   # alternating: drift of clocks or neighbours hits every arm alike
            t0 = time.perf_counter()
            idx = build()
            build_s[name].append(time.perf_counter() - t0)
            device_bytes[name] = int(idx.info().device_bytes)
            if rnd == 0:
                r = idx.search_batch(q_off, q_terms, k)
                if ref is None:
                    ref = r
                identical[name] = all(np.array_equal(r[key], ref[key]) for key in ("doc", "score", "score64", "n"))
            idx.close()
            del idx
    result = {"metric": "build wall time from stored blocks (s), sharded and unsharded, C3 corpus",
              "workload": f"C3: {c.n_docs} docs, vocab {vocab} uniform, 128 terms/doc, {int(c.n_postings)} postings, "
                          f"{int(eb.n_blocks)} stored blocks, {int(eb.n_bytes)} payload bytes; rows checked on {nq} "
                          f"3-term queries, top-{k}",
              "rounds": a.rounds, "card": card(), "gen_s": round(t_gen, 1), "encode_s": round(t_enc, 1),
              "arms": {name: {"build_s_median": round(statistics.median(build_s[name]), 3),
                              "build_s_min": round(min(build_s[name]), 3), "device_bytes": device_bytes[name],
                              "identical_rows": identical[name]} for name in arms},
              "note": "one arm resident at a time; build wall time includes the host-side checks and gathers"}
    print(json.dumps(result))
    if not all(identical.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
