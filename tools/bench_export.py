#!/usr/bin/env python
"""bench_export.py — what writing a sealed index out as the reference's stored segment costs on the GPU
(bm25x_index_export_blocks) next to the oracle's scalar encoder of the same codec on the host (orc_encode_blocks).

Corpus: C3 of bench.py (its seeds: 10M documents, vocabulary 100k, 128 terms each).  Alternating the two arms round by
round, the median of:
  export_ms   Index.export_blocks end to end (sizing call, allocation, export; host clock, the call ends in a synchronize)
  host_ms     oracle.EncodedBlocks over the same CSR (orc_encode_blocks: sizing pass + encode pass, one thread)
and, as the third arm of every round, one more export under torch.profiler (CUDA activities: the device timestamps CUPTI
records for each kernel and copy; the export runs on the library's own stream, out of reach of events a caller records),
whose device time of the export kernels (k_export_dir, k_export_tokens, k_export_encode) and of its device-to-host
copies is taken per round, median over the rounds.  The export must equal the host
encoder's payloads and directory byte for byte, and from_blocks(export) must answer `--queries` 3-term top-10 queries
with the same rows as the index itself.  Prints one JSON line with the card's name and power limit, read in the same run;
writes nothing.

  python tools/bench_export.py [--rounds 3] [--docs N] [--queries Q]
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


def ms(f):
    t0 = time.perf_counter()
    r = f()
    return (time.perf_counter() - t0) * 1e3, r


def profiled(ix):
    """Device time (ms) of the export's kernels (per kernel) and of its D2H copies, from one profiled export."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ix.export_blocks()
        torch.cuda.synchronize()
    kern, copy = {}, 0.0
    for ev in prof.events():
        name, dur = ev.name, ev.device_time_total / 1e3
        k = next((k for k in ("k_export_dir", "k_export_tokens", "k_export_encode") if k in name), None)
        if k:
            kern[k] = kern.get(k, 0.0) + dur
        elif "Memcpy DtoH" in name or "Memcpy D2H" in name:
            copy += dur
    return kern, copy


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    a = ap.parse_args()
    import _pkg
    from oracle import oracle as orc
    m = _pkg.load()
    m.load_library()
    seed, vocab = 0xB25C0DE0 + 3, 100_000
    c = m.synth_corpus(seed, a.docs, vocab, 128)
    ix = m.Index.from_corpus(c)
    oc = orc.Corpus(c.n_docs, c.doc_len, c.n_terms, c.post_off, c.post_doc, c.post_tf)
    ix.export_blocks()                      # warm-up: module load, first allocations
    t_exp, t_host, kerns, copies = [], [], [], []
    got = eb = None
    for _ in range(a.rounds):
        t, got = ms(lambda: ix.export_blocks())
        t_exp.append(t)
        got = None
        t, eb = ms(lambda: orc.EncodedBlocks(oc))
        t_host.append(t)
        kern, copy = profiled(ix)
        kerns.append(kern)
        copies.append(copy)
    args, extra = ix.export_blocks()
    nb = eb.n_blocks
    same = (args["data"].tobytes() == eb.bytes[:eb.n_bytes].tobytes() and
            all(np.array_equal(args[k], v[:nb]) for k, v in (("blk_min_doc", eb.blk_min), ("blk_n", eb.blk_n),
                                                             ("blk_meta_doc", eb.meta_doc), ("blk_meta_tf", eb.meta_tf),
                                                             ("blk_doc_off", eb.doc_off), ("blk_tf_off", eb.tf_off))) and
            np.array_equal(args["term_blk_off"], eb.term_blk_off))
    back = m.Index.from_blocks(**args)
    q_off, q_terms = m.synth_queries(seed + 1000, a.queries, vocab, 3, 3, c.post_off)
    r0, r1 = ix.search_batch(q_off, q_terms, 10), back.search_batch(q_off, q_terms, 10)
    rows_equal = all(np.array_equal(r0[k], r1[k]) for k in ("doc", "score", "score64", "n"))
    back.close()
    kern = {k: statistics.median(r.get(k, 0.0) for r in kerns) for k in kerns[0]}
    dev = statistics.median(sum(r.values()) for r in kerns)
    print(json.dumps({
        "bench": "export", "docs": a.docs, "n_blocks": nb, "payload_bytes": eb.n_bytes, "rounds": a.rounds,
        "export_ms": round(statistics.median(t_exp), 1), "host_encode_ms": round(statistics.median(t_host), 1),
        "export_ms_all": [round(x, 1) for x in t_exp], "host_encode_ms_all": [round(x, 1) for x in t_host],
        "device_kernel_ms": {k: round(v, 2) for k, v in kern.items()}, "device_kernels_total_ms": round(dev, 2),
        "device_d2h_ms": round(statistics.median(copies), 1), "device_d2h_ms_all": [round(x, 1) for x in copies],
        "bytes_equal_host_encoder": bool(same), "round_trip_rows_equal": bool(rows_equal), "card": card()}))
    ix.close()
    if not (same and rows_equal):
        sys.exit(1)


if __name__ == "__main__":
    main()
